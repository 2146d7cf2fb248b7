"""Host-side operators: thin, allocation-only wrappers that turn torch tensors into C-ABI calls.

PyTorch here is plumbing (device memory, streams, RNG); every FLOP of the sampling path runs in libb200gen.so.
Internal activation format: :class:`CL` — channels-last h16 ``[N, D, H, W, pitch]`` (2-D images have D == 1),
``pitch`` = channels rounded up to 8 (the 16-byte TMA stride granule).
"""
from __future__ import annotations

import ctypes as C
import numbers
import struct
import weakref
from dataclasses import dataclass
from typing import Sequence

import torch

from . import _lib
from ._lib import (ACT_GEGLU, ACT_GELU, ACT_LEAKYRELU, ACT_LEAKYRELU02, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SILU, ACT_TANH, DT_H16, DT_F32, DdimCoef, DdpmCoef, GnApplyParams, GnStatsParams,
                   IgemmParams, PndmCoef, check)

# torch dtype of the library's 16-bit storage type (fp16 unless B200_ACT_DTYPE=h16; see _lib.ACT_DTYPE)
H16 = torch.float16 if _lib.ACT_DTYPE == "fp16" else torch.bfloat16

__all__ = ["CL", "to_cl", "from_cl", "PackedConv", "PackedConvTranspose", "PackedLinear", "conv", "conv_transpose",
           "linear", "linear_geglu", "fork", "groupnorm", "layernorm", "upsample_nearest2x", "avgpool2", "axpy", "geglu", "attention",
           "timestep_embedding", "small_linear", "ACT_NONE", "ACT_RELU", "ACT_SILU", "ACT_LEAKYRELU", "ACT_GELU", "ACT_TANH", "ACT_SIGMOID",
           "ACT_LEAKYRELU02", "upsample2x_interp", "vae_reparam_kld", "pool_s2", "batchnorm_fold", "interpolate",
           "interpolate_plan"]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


_SIDE_STREAMS: dict = {}


class fork:
    """Run an independent branch on a side stream WHILE THE CURRENT STREAM IS BEING CAPTURED, so that a CUDA-graph replay
    executes it concurrently with what the main stream does next (a latent-UNet step is a chain of ~150 dependent
    kernels of 5-10 us; the 1x1 skip convolution of a ResnetBlock and the V^T projection of an attention block do not
    depend on their neighbours).  Outside a capture it is a no-op (the eager path is host-bound; events would only add
    to it).  Outputs the main stream reads later must be allocated BEFORE the fork (main-stream ordered frees).

        with ops.fork() as f:
            side_result = <launches>          # on the side stream when capturing
        <main-stream launches>
        f.join()                              # main waits for the branch
    """

    def __enter__(self):
        self.active = torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()
        if self.active:
            self.main = torch.cuda.current_stream()
            idx = self.main.device.index
            side = _SIDE_STREAMS.get(idx)
            if side is None:
                side = _SIDE_STREAMS[idx] = torch.cuda.Stream(device=self.main.device)
            side.wait_stream(self.main)
            self.side = side
            self._ctx = torch.cuda.stream(side)
            self._ctx.__enter__()
        return self

    def __exit__(self, *exc):
        if self.active:
            self._ctx.__exit__(*exc)
        return False

    def join(self) -> None:
        if self.active:
            self.main.wait_stream(self.side)
            self.active = False


def _ptr(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


@dataclass
class CL:
    """Channels-last h16 activation: ``t`` is ``[N, D, H, W, pitch]`` contiguous, ``C`` valid channels."""
    t: torch.Tensor
    C: int
    spatial_dims: int = 2
    # GroupNorm partial sums the producing convolution left behind: fp32 [N, slots, C/8, 2] (see b200_igemm gn_partial)
    gn: torch.Tensor | None = None

    @property
    def N(self) -> int: return self.t.shape[0]
    @property
    def D(self) -> int: return self.t.shape[1]
    @property
    def H(self) -> int: return self.t.shape[2]
    @property
    def W(self) -> int: return self.t.shape[3]
    @property
    def pitch(self) -> int: return self.t.shape[4]
    @property
    def spatial(self) -> int: return self.t.shape[1] * self.t.shape[2] * self.t.shape[3]

    def like(self, C_: int | None = None, dims: Sequence[int] | None = None) -> "CL":
        C_ = self.C if C_ is None else C_
        d = (self.D, self.H, self.W) if dims is None else tuple(dims)
        t = torch.empty((self.N, *d, round_up(C_, 8)), dtype=H16, device=self.t.device)
        return CL(t, C_, self.spatial_dims)


def new_cl(N: int, dims: Sequence[int], C_: int, device, spatial_dims: int) -> CL:
    t = torch.empty((N, *dims, round_up(C_, 8)), dtype=H16, device=device)
    return CL(t, C_, spatial_dims)


# --------------------------------------------------------------------------------------------------
# API-edge layout conversion
# --------------------------------------------------------------------------------------------------
def to_cl(x: torch.Tensor) -> CL:
    """NC[D]HW float tensor -> channels-last h16 (pad channels zero)."""
    lib = _lib.require_device()
    if x.dim() not in (4, 5):
        raise ValueError(f"expected a 4-D or 5-D NC[D]HW tensor, got shape {tuple(x.shape)}")
    sd = x.dim() - 2
    x = x.contiguous().float()
    N, C_ = x.shape[0], x.shape[1]
    dims = (1, *x.shape[2:]) if sd == 2 else tuple(x.shape[2:])
    out = new_cl(N, dims, C_, x.device, sd)
    sp = dims[0] * dims[1] * dims[2]
    check(lib.b200_nchw_to_nhwc(x.data_ptr(), N, C_, sp, out.t.data_ptr(), out.pitch, _stream()), "b200_nchw_to_nhwc")
    return out


def from_cl(a: CL, dtype=torch.float32) -> torch.Tensor:
    lib = _lib.require_device()
    shape = (a.N, a.C, a.H, a.W) if a.spatial_dims == 2 else (a.N, a.C, a.D, a.H, a.W)
    y = torch.empty(shape, dtype=torch.float32, device=a.t.device)
    check(lib.b200_nhwc_to_nchw(a.t.data_ptr(), DT_H16, a.N, a.C, a.spatial, a.pitch, y.data_ptr(), _stream()),
          "b200_nhwc_to_nchw")
    return y if dtype == torch.float32 else y.to(dtype)


def from_cl_f32(t: torch.Tensor, C_: int, spatial_dims: int) -> torch.Tensor:
    """fp32 channels-last [N, D, H, W, pitch] -> NC[D]HW fp32."""
    lib = _lib.require_device()
    N, D, H, W, P = t.shape
    shape = (N, C_, H, W) if spatial_dims == 2 else (N, C_, D, H, W)
    y = torch.empty(shape, dtype=torch.float32, device=t.device)
    check(lib.b200_nhwc_to_nchw(t.data_ptr(), DT_F32, N, C_, D * H * W, P, y.data_ptr(), _stream()), "b200_nhwc_to_nchw")
    return y


# --------------------------------------------------------------------------------------------------
# weight packing (one-time, cached by the modules; not on the per-step path)
# --------------------------------------------------------------------------------------------------
def _src_f32(weight: torch.Tensor) -> torch.Tensor:
    w = weight.detach()
    return w if (w.dtype == torch.float32 and w.is_contiguous()) else w.float().contiguous()


def repack(w: torch.Tensor, cout: int, cin: int, taps: int, blocks, rows: int, *, transposed: bool = False,
           mode: int = _lib.REPACK_BLOCKS, pitch: int | None = None) -> torch.Tensor:
    """One b200_repack_weight launch: fp32 parameter ``w`` -> K-major h16 ``[round_up(rows, 16), pitch]``.
    ``blocks`` = [(cin0, cs, (tap, ...)), ...] in segment order; every block is ceil64(cs) columns wide."""
    lib = _lib.require_device()
    arr, col = None, 0
    if mode == _lib.REPACK_BLOCKS:
        arr = (_lib.RepackBlock * len(blocks))()
        for i, (cin0, cs, taps_i) in enumerate(blocks):
            b = arr[i]
            b.col0, b.cin0, b.cs, b.ntaps = col, cin0, cs, len(taps_i)
            for j, t in enumerate(taps_i):
                b.tap[j] = t
            col += round_up(cs, 64)
        pitch = col
    out = torch.empty((round_up(rows, 16), pitch), dtype=H16, device=w.device)
    check(lib.b200_repack_weight(w.data_ptr(), cout, cin, taps, int(transposed), mode, arr, len(blocks) if blocks else 0,
                                 out.data_ptr(), out.shape[0], pitch, _stream()), "b200_repack_weight")
    return out


class PackedConv:
    """K-major h16 weight matrix + tap table for one nn.Conv{2,3}d.

    ``splits`` are the channel counts of the (up to two) input tensors the conv reads — the virtual concat of
    the UNet up path.  ``padding`` is ``(lo, hi)`` per spatial dim (asymmetric for the AutoencoderKL downsampler,
    autoencoderkl.py:107-120).
    """

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor | None, stride: int | Sequence[int],
                 padding, splits: Sequence[int] | None = None):
        w = _src_f32(weight)
        sd = w.dim() - 2
        self.spatial_dims = sd
        self.cout, cin = w.shape[0], w.shape[1]
        k = tuple(w.shape[2:])
        if sd == 2:
            k = (1, *k)
        self.k = k
        st = (stride,) * sd if isinstance(stride, int) else tuple(stride)
        self.stride = (1, *st) if sd == 2 else st
        if isinstance(padding, int):
            padding = [(padding, padding)] * sd
        padding = [(p, p) if isinstance(p, int) else tuple(p) for p in padding]
        self.pad = [(0, 0), *padding] if sd == 2 else padding
        self.splits = list(splits) if splits else [cin]
        if sum(self.splits) != cin or len(self.splits) > 2:
            raise ValueError(f"channel splits {self.splits} do not match weight in_channels {cin}")
        blocks, segs = [], []
        for a in range(k[0]):
            for b in range(k[1]):
                for c in range(k[2]):
                    off = 0
                    for s, cs in enumerate(self.splits):
                        blocks.append((off, cs, ((a * k[1] + b) * k[2] + c,)))
                        segs.append((s, c - self.pad[2][0], b - self.pad[1][0], a - self.pad[0][0], 0,
                                     round_up(cs, 64) // 64))
                        off += cs
        if len(segs) > _lib.IGEMM_MAX_SEG:
            raise ValueError(f"convolution needs {len(segs)} taps; the kernel supports {_lib.IGEMM_MAX_SEG}")
        taps = k[0] * k[1] * k[2]
        self.w = repack(w, self.cout, cin, taps, blocks, self.cout)
        self.segs = segs
        self.bias = None if bias is None else _src_f32(bias)
        # Degenerate ends of the UNet (see b200_tap_gather / b200_tap_sum): with very few input channels the taps
        # are folded into ONE 64-wide K chunk; with very few output channels the taps become GEMM columns.
        self.tap_in = self.tap_out = None
        if taps > 1 and len(self.splits) == 1 and taps * cin <= 64:
            # [co][tap*cin + c]
            self.tap_in = PackedLinear.from_packed(repack(w, self.cout, cin, taps, None, self.cout,
                                                          mode=_lib.REPACK_TAP_IN, pitch=64),
                                                   self.cout, taps * cin, self.bias)
        elif (taps > 1 and len(self.splits) == 1 and self.cout <= 4 and taps * self.cout <= 128 and cin >= 64
              and self.stride == (1, 1, 1)):
            # [tap*cout + co][c]; the GEMM's column count is rounded up to 32 (zero rows): full 32-column chunks take
            # the vectorised epilogue (27 columns would go through the much slower per-element path)
            ncol = round_up(taps * self.cout, 32)
            self.tap_out = PackedLinear.from_packed(repack(w, self.cout, cin, taps, None, ncol,
                                                           mode=_lib.REPACK_TAP_OUT, pitch=round_up(cin, 64)),
                                                    ncol, cin, None)

    def geom(self, N: int, D: int, H: int, W: int):
        od = self.out_dims(D, H, W)
        return (C.c_int32 * 16)(N, D, H, W, *od, *self.k, *self.stride, self.pad[0][0], self.pad[1][0], self.pad[2][0])

    def out_dims(self, D: int, H: int, W: int) -> tuple[int, int, int]:
        i = (D, H, W)
        return tuple((i[d] + self.pad[d][0] + self.pad[d][1] - self.k[d]) // self.stride[d] + 1 for d in range(3))


class PackedLinear:
    """nn.Linear weight [O, K] -> K-major h16 (already K-major; only padded and cast)."""

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor | None):
        w = _src_f32(weight)
        self.cout, self.K = w.shape
        self.w = repack(w, self.cout, self.K, 1, [(0, self.K, (0,))], self.cout)
        self.segs = [(0, 0, 0, 0, 0, round_up(self.K, 64) // 64)]
        self.bias = None if bias is None else _src_f32(bias)
        self.stride = (1, 1, 1)

    @classmethod
    def stacked(cls, weights, biases) -> "PackedLinear":
        """Several nn.Linear layers with the same input applied as ONE GEMM: their weight matrices stacked along the
        output dimension (each repacked by its own launch into its row range of one matrix).  Every layer but the
        last must have a multiple of 16 output features (the packed row granule)."""
        ws = [_src_f32(w) for w in weights]
        K = ws[0].shape[1]
        outs = [w.shape[0] for w in ws]
        if any(w.shape[1] != K for w in ws) or any(o % 16 for o in outs[:-1]):
            raise ValueError("stacked linears need a common input width and 16-row-aligned blocks")
        lib = _lib.require_device()
        pitch = round_up(K, 64)
        w16 = torch.empty((round_up(sum(outs), 16), pitch), dtype=H16, device=ws[0].device)
        blk = (_lib.RepackBlock * 1)()
        blk[0].col0, blk[0].cin0, blk[0].cs, blk[0].ntaps = 0, 0, K, 1
        row = 0
        for w, o in zip(ws, outs):
            rows_pad = round_up(o, 16)
            check(lib.b200_repack_weight(w.data_ptr(), o, K, 1, 0, _lib.REPACK_BLOCKS, blk, 1,
                                         w16.data_ptr() + row * pitch * 2, rows_pad, pitch, _stream()),
                  "b200_repack_weight")
            row += o
        bias = None
        if any(b is not None for b in biases):
            bias = torch.cat([(_src_f32(b) if b is not None else torch.zeros(o, device=ws[0].device))
                              for b, o in zip(biases, outs)]).contiguous()
        return cls.from_packed(w16, sum(outs), K, bias)

    @classmethod
    def geglu(cls, weight: torch.Tensor, bias: torch.Tensor | None) -> "PackedLinear":
        """linear1 of a GEGLU feed-forward (weight [2H, K]: rows [0, H) = a, [H, 2H) = gate; monai MLPBlock
        act="GEGLU") with its rows — and bias — interleaved in groups of 32 ([32 a | 32 gate] per 64 GEMM columns), the
        layout b200_igemm's B200_ACT_GEGLU epilogue gates in place.  H must be a multiple of 32."""
        w = _src_f32(weight)
        H = w.shape[0] // 2
        if w.shape[0] != 2 * H or H % 32:
            raise ValueError(f"GEGLU linear needs 2 x (multiple of 32) output features, got {w.shape[0]}")
        j = torch.arange(2 * H, device=w.device)
        perm = (j // 64) * 32 + (j % 32) + ((j % 64) // 32) * H          # GEMM column -> source row
        self = cls(w.index_select(0, perm), None if bias is None else _src_f32(bias).index_select(0, perm))
        self.geglu_hidden = H
        return self

    @classmethod
    def from_packed(cls, w16: torch.Tensor, cout: int, K: int, bias: torch.Tensor | None) -> "PackedLinear":
        self = cls.__new__(cls)
        self.cout, self.K, self.w = cout, K, w16
        self.segs = [(0, 0, 0, 0, 0, round_up(K, 64) // 64)]
        self.bias, self.stride = bias, (1, 1, 1)
        return self


class PackedConvTranspose:
    """nn.ConvTranspose{2,3}d as one stride-1 implicit GEMM per output phase (out = i*s - p + k)."""

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor | None, stride: int, padding: int,
                 output_padding: int):
        w = _src_f32(weight)                  # [Cin, Cout, k...]
        sd = w.dim() - 2
        self.spatial_dims = sd
        self.cin, self.cout = w.shape[0], w.shape[1]
        k = tuple(w.shape[2:])
        if sd == 2:
            k = (1, *k)
        self.k = k
        self.s = (1, stride, stride) if sd == 2 else (stride,) * 3
        self.p = (0, padding, padding) if sd == 2 else (padding,) * 3
        self.op = (0, output_padding, output_padding) if sd == 2 else (output_padding,) * 3
        self.bias = None if bias is None else _src_f32(bias)
        nch = round_up(self.cin, 64) // 64
        ntaps = k[0] * k[1] * k[2]
        self.phases = []
        for rd in range(self.s[0]):
            for rh in range(self.s[1]):
                for rw in range(self.s[2]):
                    r = (rd, rh, rw)
                    taps = [[(kk, (r[d] + self.p[d] - kk) // self.s[d]) for kk in range(k[d])
                             if (r[d] + self.p[d] - kk) % self.s[d] == 0] for d in range(3)]
                    blocks, segs = [], []
                    for (a, oa) in taps[0]:
                        for (b, ob) in taps[1]:
                            for (c, oc) in taps[2]:
                                blocks.append((0, self.cin, ((a * k[1] + b) * k[2] + c,)))
                                segs.append((0, oc, ob, oa, 0, nch))
                    if not segs:
                        continue
                    self.phases.append((r, repack(w, self.cout, self.cin, ntaps, blocks, self.cout, transposed=True),
                                        segs))

    def out_dims(self, D: int, H: int, W: int) -> tuple[int, int, int]:
        i = (D, H, W)
        return tuple((i[d] - 1) * self.s[d] - 2 * self.p[d] + self.k[d] + self.op[d] for d in range(3))


class PackedUpsampleConv:
    """nearest x2 upsample followed by a k3 p1 convolution (Upsample blocks, diffusion_model_unet.py:574-586,
    autoencoderkl.py:79-93) WITHOUT materialising the 4x/8x larger tensor: for each output phase (o = 2i + p per
    dim) the three taps read only two distinct input voxels, so the op is 4 (2-D) / 8 (3-D) stride-1 convolutions
    with 2-tap kernels on the low-resolution input whose weights are sums of the original taps
        p = 0:  in[i-1] * w0 + in[i] * (w1 + w2)         p = 1:  in[i] * (w0 + w1) + in[i+1] * w2
    each writing its phase of the output with doubled strides.  27 -> 8 taps per output voxel (3.4x fewer FLOPs).
    Zero padding of the upsampled tensor maps to the TMA zero fill at in[-1] / in[n]."""

    _TAPS = {0: ((-1, (0,)), (0, (1, 2))), 1: ((0, (0, 1)), (1, (2,)))}

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor | None):
        w = _src_f32(weight)
        sd = w.dim() - 2
        if tuple(w.shape[2:]) != (3,) * sd:
            raise ValueError("PackedUpsampleConv expects a 3^d kernel")
        self.spatial_dims = sd
        self.cout, self.cin = w.shape[0], w.shape[1]
        kk = (1, 3, 3) if sd == 2 else (3, 3, 3)
        self.bias = None if bias is None else _src_f32(bias)
        nch = round_up(self.cin, 64) // 64
        self.phases = []
        d_phases = (0, 1) if sd == 3 else (None,)
        for pd in d_phases:
            for ph in (0, 1):
                for pw in (0, 1):
                    td = self._TAPS[pd] if pd is not None else ((0, (0,)),)
                    blocks, segs = [], []
                    for (od, kds) in td:
                        for (oh, khs) in self._TAPS[ph]:
                            for (ow, kws) in self._TAPS[pw]:
                                src_taps = tuple((a * kk[1] + b) * kk[2] + c for a in kds for b in khs for c in kws)
                                blocks.append((0, self.cin, src_taps))
                                segs.append((0, ow, oh, od, 0, nch))
                    self.phases.append(((pd or 0, ph, pw), repack(w, self.cout, self.cin, kk[0] * kk[1] * kk[2],
                                                                   blocks, self.cout), segs))


def conv_upsample2x(src: CL, pu: PackedUpsampleConv, impl: int = 0) -> CL:
    sd = src.spatial_dims
    od = (src.D * 2 if sd == 3 else src.D, src.H * 2, src.W * 2)
    out = new_cl(src.N, od, pu.cout, src.t.device, sd)
    P = out.pitch
    full = (od[0] * od[1] * od[2] * P, od[1] * od[2] * P, od[2] * P, P)
    sdd = 2 if sd == 3 else 1
    part = _gn_partial_for(out, src.N * src.D * src.H * src.W, 8, launches=len(pu.phases))
    for i, (r, w, segs) in enumerate(pu.phases):
        off = r[0] * full[1] + r[1] * full[2] + r[2] * full[3]
        strides = (full[0], full[1] * sdd, full[2] * 2, full[3] * 2)
        p = _conv_params([src], w, segs, (1, 1, 1), out.t, (src.D, src.H, src.W), pu.cout, DT_H16, pu.bias, None,
                         ACT_NONE, 1.0, None, DT_H16, ACT_NONE, out_elem_off=off, out_strides=strides, impl=impl)
        if part is not None:          # every phase launch owns its own range of slots
            p.gn_partial, p.gn_slots, p.gn_slot0 = part.data_ptr(), part.shape[1], i * _gn_slots()
            p.gn_group = _gn_group(out)
        igemm_raw(p)
    return out


_TAP_MIN_ROWS = 1 << 15       # below this the extra launch costs more than the padded implicit GEMM
_GN_FUSE_MIN_ROWS = 1 << 15   # below this a separate statistics pass is cheaper than the zero-fill + wider reduce
_GN_FUSE = True
_SM_COUNT = None


def _gn_slots(launches: int = 1) -> int:
    global _SM_COUNT
    if _SM_COUNT is None:
        _SM_COUNT = int(_lib.require_device().b200_sm_count())
    return 4 * _SM_COUNT * launches


def _gn_partial_for(out: CL, rows: int, n_seg: int, launches: int = 1) -> torch.Tensor | None:
    """Zero-filled partial-sum buffer if this output is worth instrumenting: a heavy (>= 8 tap) convolution writing a
    large h16 tensor whose channel count tiles the 32-column epilogue chunks."""
    if not _GN_FUSE or rows < _GN_FUSE_MIN_ROWS or n_seg < 8 or out.C % 32 != 0 or out.pitch != out.C:
        return None
    # partial groups of 8 channels; of 4 for narrow tensors, whose GroupNorm(32) groups are 4 channels wide (128 channels:
    # level 0 of the 2-D UNets, the AutoencoderKL) — the consumer reads the width off the buffer's shape
    gw = 4 if out.C <= 128 else 8
    out.gn = torch.zeros((out.N, _gn_slots(launches), out.C // gw, 2), dtype=torch.float32, device=out.t.device)
    return out.gn


def _gn_group(a: CL) -> int:
    return a.C // a.gn.shape[2]


# --------------------------------------------------------------------------------------------------
# implicit GEMM launcher
# --------------------------------------------------------------------------------------------------
# id(packed weight tensor) -> (weakref to it, segs, IgemmParams with weight + tap table filled).  Weak: the cache must not
# keep the packed weights of a deleted model alive (round-1 review); a dead or recycled id simply misses.
_PARAM_TEMPLATES: dict = {}


def _fill_segs(p: IgemmParams, segs) -> None:
    p.n_seg = len(segs)
    for i, (src, dw, dh, dd, c0, nch) in enumerate(segs):
        s = p.seg[i]
        s.src, s.dw, s.dh, s.dd, s.c0, s.nchunks = src, dw, dh, dd, c0, nch


_SPLIT_K = True          # tests and probes set it to False to compare split and one-pass reductions
_SPLIT_LAUNCHES = 0      # calls that went through the split-K pair of kernels (tests / probes read it)


def igemm_raw(p: IgemmParams, split_k: bool = True) -> None:
    """One b200_igemm launch.  Calls whose grid cannot fill the SMs (deep levels of a latent UNet, single-sample
    linears) get the split-K workspace the library asks for; everything else is a single kernel.  ``split_k=False``
    keeps every call one pass, so a row's result does not depend on how many other rows the call has."""
    lib = _lib.require_device()
    ws = None
    if _SPLIT_K and split_k and not p.split_ws:
        need = int(lib.b200_igemm_split_workspace_bytes(C.byref(p)))
        if need:
            global _SPLIT_LAUNCHES
            _SPLIT_LAUNCHES += 1
            dev = torch.device("cuda", torch.cuda.current_device())
            ws = torch.empty(need, dtype=torch.uint8, device=dev)
            p.split_ws, p.split_ws_bytes = ws.data_ptr(), need
    try:
        check(lib.b200_igemm(C.byref(p), _stream()), "b200_igemm")
    finally:
        if ws is not None:       # the struct may be a cached template: never keep the pointers
            p.split_ws, p.split_ws_bytes = None, 0


def _conv_params(srcs: Sequence[CL], w: torch.Tensor, segs, stride, out_t: torch.Tensor, out_dims, cout: int,
                 out_dtype: int, bias, rowvec, act1: int, scale: float, res: torch.Tensor | None, res_dtype: int,
                 act2: int, out_elem_off: int = 0, out_strides=None, res_strides=None, impl: int = 0) -> IgemmParams:
    # the tap table (up to 128 segments), weight pointer and stride are fixed for a packed weight: filling them
    # field by field through ctypes costs ~30 us per 27-tap call, a struct copy of a per-weight template 0.5 us
    tmpl = _PARAM_TEMPLATES.get(id(w))
    if tmpl is not None and tmpl[0]() is w and tmpl[1] is segs:
        p = IgemmParams.from_buffer_copy(tmpl[2])
    else:
        p = IgemmParams()
        p.w_ptr = w.data_ptr()
        p.w_rows, p.w_pitch, p.w_K = w.shape[0], w.shape[1], 0
        p.w_bstride, p.w_batched = 0, 0
        _fill_segs(p, segs)
        if len(_PARAM_TEMPLATES) > 4096:
            _PARAM_TEMPLATES.clear()
        key = id(w)
        _PARAM_TEMPLATES[key] = (weakref.ref(w, lambda _r, _k=key: _PARAM_TEMPLATES.pop(_k, None)), segs,
                                 IgemmParams.from_buffer_copy(p))
    a0 = srcs[0]
    for i, a in enumerate(srcs):
        if (a.N, a.D, a.H, a.W) != (a0.N, a0.D, a0.H, a0.W):
            raise ValueError("concatenated inputs must share batch and spatial extent")
        p.a_ptr[i] = a.t.data_ptr()
        p.a_C[i] = a.C
        p.a_pitch[i] = a.pitch
    p.in_N, p.in_D, p.in_H, p.in_W = a0.N, a0.D, a0.H, a0.W
    p.stride_d, p.stride_h, p.stride_w = stride
    esz = 2 if out_dtype == DT_H16 else 4
    p.out_ptr = out_t.data_ptr() + out_elem_off * esz
    p.out_dtype = out_dtype
    p.out_N = a0.N
    p.out_D, p.out_H, p.out_W = out_dims
    P = out_t.shape[-1]
    p.cout, p.out_cols = cout, P
    if out_strides is None:
        OD, OH, OW = out_t.shape[1:4]
        out_strides = (OD * OH * OW * P, OH * OW * P, OW * P, P)
    p.out_sN, p.out_sD, p.out_sH, p.out_sW = out_strides
    p.bias = _ptr(bias)
    if rowvec is not None:
        p.rowvec = rowvec.data_ptr()
        p.rowvec_bstride = rowvec.stride(0) if rowvec.shape[0] > 1 else 0
    p.act1, p.scale, p.act2 = act1, scale, act2
    if res is not None:
        p.res_ptr = res.data_ptr() + (out_elem_off * (2 if res_dtype == DT_H16 else 4))
        p.res_dtype = res_dtype
        if res_strides is None:
            RP = res.shape[-1]
            RD, RH, RW = res.shape[1:4]
            res_strides = (RD * RH * RW * RP, RH * RW * RP, RW * RP, RP)
        p.res_sN, p.res_sD, p.res_sH, p.res_sW = res_strides
    p.impl = impl
    return p


def conv(srcs: CL | Sequence[CL], pc: PackedConv, *, rowvec: torch.Tensor | None = None, act1: int = ACT_NONE,
         scale: float = 1.0, residual: CL | None = None, act2: int = ACT_NONE, out_f32: bool = False,
         impl: int = 0, out: CL | None = None, gn_stats: bool = True, split_k: bool = True) -> CL | torch.Tensor:
    """Fused convolution: act2(residual + scale * act1(conv(cat(srcs)) + bias + rowvec[n])).

    Returns a :class:`CL` (h16) or, with ``out_f32``, an fp32 channels-last tensor ``[N, D, H, W, round_up(C, 4)]``.
    ``gn_stats=False`` skips the GroupNorm partial sums for an output no GroupNorm reads; ``split_k``: igemm_raw.
    """
    if isinstance(srcs, CL):
        srcs = [srcs]
    if [a.C for a in srcs] != pc.splits:
        raise ValueError(f"conv inputs have channels {[a.C for a in srcs]} but weights were packed for {pc.splits}")
    a0 = srcs[0]
    od = pc.out_dims(a0.D, a0.H, a0.W)
    if min(od) < 1:
        raise ValueError(f"convolution output would be empty for input {(a0.D, a0.H, a0.W)}")
    if out_f32:
        out_t = torch.empty((a0.N, *od, round_up(pc.cout, 4)), dtype=torch.float32, device=a0.t.device)
        out = out_t
    else:
        if out is None:
            out = new_cl(a0.N, od, pc.cout, a0.t.device, a0.spatial_dims)
        elif tuple(out.t.shape[:4]) != (a0.N, *od) or out.C != pc.cout:
            raise ValueError("preallocated convolution output has the wrong shape")
        out_t = out.t
    if residual is not None and tuple(residual.t.shape[:4]) != tuple(out_t.shape[:4]):
        raise ValueError("residual shape mismatch")
    rows = a0.N * od[0] * od[1] * od[2]
    if impl == 0 and rows >= _TAP_MIN_ROWS and pc.tap_in is not None:
        # conv_in-like: im2col of the few input channels (one h16 row of <= 64 values per output voxel), then the
        # ordinary fused GEMM epilogue
        x2 = tap_gather(a0, pc.geom(a0.N, a0.D, a0.H, a0.W), pc.k[0] * pc.k[1] * pc.k[2])
        pl = pc.tap_in
        p = _conv_params([x2], pl.w, pl.segs, (1, 1, 1), out_t, od, pc.cout,
                         DT_F32 if out_f32 else DT_H16, pl.bias, rowvec, act1, scale,
                         None if residual is None else residual.t, DT_H16, act2)
        igemm_raw(p)
        return out
    if (impl == 0 and rows >= _TAP_MIN_ROWS and pc.tap_out is not None and rowvec is None and residual is None
            and act1 == ACT_NONE and act2 == ACT_NONE and scale == 1.0):
        # out-conv-like: Y[v][tap*cout+co] = x[v] . w[co, :, tap] reads x once; the taps are summed afterwards
        lib = _lib.require_device()
        y = linear(a0, pc.tap_out, out_f32=True)
        check(lib.b200_tap_sum(y.data_ptr(), y.shape[-1], pc.geom(a0.N, a0.D, a0.H, a0.W), pc.cout, _ptr(pc.bias),
                               out_t.data_ptr(), out_t.shape[-1], DT_F32 if out_f32 else DT_H16, _stream()),
              "b200_tap_sum")
        return out
    p = _conv_params(srcs, pc.w, pc.segs, pc.stride, out_t, od, pc.cout, DT_F32 if out_f32 else DT_H16, pc.bias,
                     rowvec, act1, scale, None if residual is None else residual.t, DT_H16, act2, impl=impl)
    if not out_f32 and gn_stats:
        part = _gn_partial_for(out, rows, len(pc.segs))
        if part is not None:
            p.gn_partial, p.gn_slots, p.gn_slot0 = part.data_ptr(), part.shape[1], 0
            p.gn_group = _gn_group(out)
    if split_k:          # the one-argument call keeps substitutes of igemm_raw(p) working
        igemm_raw(p)
    else:
        igemm_raw(p, split_k=False)
    return out


def conv_transpose(src: CL, pt: PackedConvTranspose, *, act1: int = ACT_NONE, impl: int = 0) -> CL:
    od = pt.out_dims(src.D, src.H, src.W)
    out = new_cl(src.N, od, pt.cout, src.t.device, src.spatial_dims)
    P = out.pitch
    full = (od[0] * od[1] * od[2] * P, od[1] * od[2] * P, od[2] * P, P)
    for (r, w, segs) in pt.phases:
        cnt = tuple((od[d] - r[d] + pt.s[d] - 1) // pt.s[d] for d in range(3))
        if min(cnt) < 1:
            continue
        off = r[0] * full[1] + r[1] * full[2] + r[2] * full[3]
        strides = (full[0], full[1] * pt.s[0], full[2] * pt.s[1], full[3] * pt.s[2])
        p = _conv_params([src], w, segs, (1, 1, 1), out.t, cnt, pt.cout, DT_H16, pt.bias, None, act1, 1.0, None,
                         DT_H16, ACT_NONE, out_elem_off=off, out_strides=strides, impl=impl)
        igemm_raw(p)
    return out


def as_rows(t: torch.Tensor, C_: int) -> CL:
    """View a h16 [..., pitch] tensor as a token matrix CL [1, 1, 1, M, pitch]."""
    P = t.shape[-1]
    return CL(t.reshape(1, 1, 1, -1, P), C_, 2)


def linear(x: CL, pl: PackedLinear, *, residual: CL | None = None, act1: int = ACT_NONE, out_f32: bool = False,
           impl: int = 0, split_k: bool = True):
    """y = x @ W^T + b over the channel dim of any CL (rows = voxels); ``split_k``: igemm_raw."""
    if x.C != pl.K:
        raise ValueError(f"linear expects {pl.K} input features, got {x.C}")
    if out_f32:
        out_t = torch.empty((*x.t.shape[:4], round_up(pl.cout, 4)), dtype=torch.float32, device=x.t.device)
        out = out_t
    else:
        out = x.like(pl.cout)
        out_t = out.t
    p = _conv_params([x], pl.w, pl.segs, (1, 1, 1), out_t, (x.D, x.H, x.W), pl.cout, DT_F32 if out_f32 else DT_H16,
                     pl.bias, None, act1, 1.0, None if residual is None else residual.t, DT_H16, ACT_NONE, impl=impl)
    if split_k:          # the one-argument call keeps substitutes of igemm_raw(p) working
        igemm_raw(p)
    else:
        igemm_raw(p, split_k=False)
    return out


def tap_gather(x: CL, geom, taps: int) -> CL:
    """b200_tap_gather: the im2col rows [N, OD, OH, OW, round_up(taps * C, 8)] of a convolution geometry ``geom``
    (PackedConv.geom's 16 values), for a GEMM over K = taps * C."""
    lib = _lib.require_device()
    K = taps * x.C
    od = tuple(geom[4:7])
    out = torch.empty((x.N, *od, round_up(K, 8)), dtype=H16, device=x.t.device)
    check(lib.b200_tap_gather(x.t.data_ptr(), x.C, x.pitch, geom, out.data_ptr(), out.shape[-1], _stream()),
          "b200_tap_gather")
    return CL(out, K, x.spatial_dims)


# --------------------------------------------------------------------------------------------------
# normalisation
# --------------------------------------------------------------------------------------------------
def _gn_params(srcs: Sequence[CL]):
    sp, ap = GnStatsParams(), GnApplyParams()
    a0 = srcs[0]
    for i, a in enumerate(srcs):
        if (a.N, a.D, a.H, a.W) != (a0.N, a0.D, a0.H, a0.W):
            raise ValueError("normalised inputs must share batch and spatial extent")
        sp.x_ptr[i] = ap.x_ptr[i] = a.t.data_ptr()
        sp.x_C[i] = ap.x_C[i] = a.C
        sp.x_pitch[i] = ap.x_pitch[i] = a.pitch
    sp.N = ap.N = a0.N
    sp.spatial = ap.spatial = a0.spatial
    return sp, ap


_ONES: dict = {}


def _const_vec(n: int, value: float, device) -> torch.Tensor:
    key = (n, value, str(device))
    if key not in _ONES:
        _ONES[key] = torch.full((n,), value, dtype=torch.float32, device=device)
    return _ONES[key]


def groupnorm_affine(srcs: CL | Sequence[CL], groups: int, eps: float, gamma: torch.Tensor | None,
                     beta: torch.Tensor | None) -> torch.Tensor:
    """Per-(sample, channel) affine table [N, C, 2] = (rstd * gamma, beta - mean * rstd * gamma) of GroupNorm over the
    virtual channel-concat of ``srcs`` (gamma / beta None = no affine, e.g. InstanceNorm with groups = C)."""
    lib = _lib.require_device()
    if isinstance(srcs, CL):
        srcs = [srcs]
    a0 = srcs[0]
    Ct = sum(a.C for a in srcs)
    if Ct % groups != 0:
        raise ValueError(f"GroupNorm: {Ct} channels not divisible by {groups} groups")
    dev = a0.t.device
    affine = torch.empty((a0.N, Ct, 2), dtype=torch.float32, device=dev)
    sp, _ = _gn_params(srcs)
    sp.groups, sp.eps = groups, eps
    g32 = _const_vec(Ct, 1.0, dev) if gamma is None else (gamma if gamma.dtype == torch.float32 else gamma.float())
    b32 = _const_vec(Ct, 0.0, dev) if beta is None else (beta if beta.dtype == torch.float32 else beta.float())
    sp.gamma, sp.beta = g32.data_ptr(), b32.data_ptr()
    sp.affine = affine.data_ptr()
    cpg = Ct // groups
    if (_GN_FUSE and all(a.gn is not None for a in srcs) and all(cpg % _gn_group(a) == 0 for a in srcs)
            and srcs[0].C % cpg == 0):
        # the producers already summed their outputs (8- or 4-channel groups) while writing them: no pass over the data
        parts = (C.c_void_p * 2)(*[a.gn.data_ptr() for a in srcs], *([None] * (2 - len(srcs))))
        slots = (C.c_int32 * 2)(*[a.gn.shape[1] for a in srcs], *([0] * (2 - len(srcs))))
        gws = (C.c_int32 * 2)(*[_gn_group(a) for a in srcs], *([0] * (2 - len(srcs))))
        check(lib.b200_groupnorm_from_partials_ex(C.byref(sp), parts, slots, gws, _stream()),
              "b200_groupnorm_from_partials_ex")
    else:
        ws = torch.empty(lib.b200_groupnorm_workspace_bytes(a0.N, a0.spatial, Ct) // 4, dtype=torch.float32, device=dev)
        sp.partial = ws.data_ptr()
        check(lib.b200_groupnorm_stats(C.byref(sp), _stream()), "b200_groupnorm_stats")
    return affine


# Single-launch GroupNorm for small tensors (b200_groupnorm_fused): one CTA per (sample, group) computes the statistics
# and applies them — GroupNorm is 138 of the 309 launches of a C2 latent-UNet step as three kernels.  Tests and probes
# set _GN_SMALL to False to compare it with the three-kernel path.
_GN_SMALL = True
_GN_SMALL_MAX_ELEMS = 1 << 17           # spatial * channels-per-group handled by one CTA


def groupnorm(srcs: CL | Sequence[CL], groups: int, eps: float, gamma: torch.Tensor, beta: torch.Tensor,
              act: int = ACT_NONE) -> CL:
    """GroupNorm (+SiLU / LeakyReLU) over the virtual channel-concat of ``srcs``; returns one dense CL."""
    lib = _lib.require_device()
    if isinstance(srcs, CL):
        srcs = [srcs]
    a0 = srcs[0]
    Ct = sum(a.C for a in srcs)
    if _GN_SMALL and Ct % groups == 0 and act in (ACT_NONE, ACT_SILU, ACT_LEAKYRELU, ACT_LEAKYRELU02):
        cpg = Ct // groups
        if a0.spatial * cpg <= _GN_SMALL_MAX_ELEMS and cpg <= 4096 and (len(srcs) == 1 or a0.C % cpg == 0) \
                and not (_GN_FUSE and all(a.gn is not None for a in srcs)):
            sp, ap = _gn_params(srcs)
            out = a0.like(Ct)
            sp.groups, sp.eps = groups, eps
            g32 = gamma if gamma.dtype == torch.float32 else gamma.float()
            b32 = beta if beta.dtype == torch.float32 else beta.float()
            sp.gamma, sp.beta = g32.data_ptr(), b32.data_ptr()
            ap.act, ap.y_ptr, ap.y_pitch = act, out.t.data_ptr(), out.pitch
            check(lib.b200_groupnorm_fused(C.byref(sp), C.byref(ap), _stream()), "b200_groupnorm_fused")
            return out
    affine = groupnorm_affine(srcs, groups, eps, gamma, beta)
    _, ap = _gn_params(srcs)
    out = a0.like(Ct)
    ap.affine, ap.act = affine.data_ptr(), act
    ap.y_ptr, ap.y_pitch = out.t.data_ptr(), out.pitch
    check(lib.b200_groupnorm_apply(C.byref(ap), _stream()), "b200_groupnorm_apply")
    return out


def spade_modulate(srcs: CL | Sequence[CL], affine: torch.Tensor, gb: CL, gb_affine: torch.Tensor,
                   act: int = ACT_NONE) -> CL:
    """act(norm(x) * (1 + inorm(gamma)) + inorm(beta)) in one pass (blocks/spade_norm.py:95): ``affine`` is the
    GroupNorm table of x, ``gb`` holds gamma | beta as channel halves, ``gb_affine`` their InstanceNorm table."""
    lib = _lib.require_device()
    if isinstance(srcs, CL):
        srcs = [srcs]
    a0 = srcs[0]
    Ct = sum(a.C for a in srcs)
    if gb.C != 2 * Ct or (gb.N, gb.D, gb.H, gb.W) != (a0.N, a0.D, a0.H, a0.W):
        raise ValueError("SPADE modulation tensor does not match the normalised input")
    _, ap = _gn_params(srcs)
    out = a0.like(Ct)
    ap.affine, ap.act = affine.data_ptr(), act
    ap.y_ptr, ap.y_pitch = out.t.data_ptr(), out.pitch
    check(lib.b200_spade_apply(C.byref(ap), gb.t.data_ptr(), gb.pitch, gb_affine.data_ptr(), _stream()),
          "b200_spade_apply")
    return out


def resize_nearest(x: CL, dims: Sequence[int]) -> CL:
    """F.interpolate(x, size=dims, mode="nearest") on a channels-last tensor."""
    d = tuple(int(v) for v in dims)
    if len(d) == 2:
        d = (1, *d)
    if d == (x.D, x.H, x.W):
        return x
    return _resample(x, d, _lib.INTERPOLATE_NEAREST)


def layernorm(x: CL, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> CL:
    lib = _lib.require_device()
    out = x.like()
    M = x.N * x.spatial
    check(lib.b200_layernorm(x.t.data_ptr(), M, x.C, x.pitch, gamma.data_ptr(), beta.data_ptr(), eps, out.t.data_ptr(),
                             out.pitch, _stream()), "b200_layernorm")
    return out


# --------------------------------------------------------------------------------------------------
# resampling / elementwise
# --------------------------------------------------------------------------------------------------
def upsample_nearest2x(x: CL) -> CL:
    """F.interpolate(x, scale_factor=2, mode="nearest"); a 2-D tensor keeps its D slices."""
    sd = x.spatial_dims
    return _resample(x, (x.D * 2 if sd == 3 else x.D, x.H * 2, x.W * 2), _lib.INTERPOLATE_NEAREST)


_INTERP_MODES = {"bilinear": _lib.INTERP_BILINEAR, "bicubic": _lib.INTERP_BICUBIC}


def upsample2x_interp(x: CL, mode: str) -> CL:
    """F.interpolate(scale_factor=2, mode="bilinear" | "bicubic", align_corners=False) of a 2-D channels-last tensor."""
    if x.spatial_dims != 2 or x.D != 1:
        raise NotImplementedError(f"{mode} x2 upsampling is 2-D only (3-D tensors take nearest)")
    if mode not in _INTERP_MODES:
        raise ValueError(f"unknown interpolation mode {mode!r}; expected one of {sorted(_INTERP_MODES)}")
    lib = _lib.require_device()
    out = x.like(dims=(1, x.H * 2, x.W * 2))
    check(lib.b200_upsample2x_interp(x.t.data_ptr(), x.N, x.H, x.W, x.pitch, _INTERP_MODES[mode], out.t.data_ptr(),
                                     _stream()), "b200_upsample2x_interp")
    return out


def vae_reparam_kld(mu: torch.Tensor, logvar: torch.Tensor, eps: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(eps * exp(0.5 * logvar) + mu, -0.5 * sum(1 + logvar - mu^2 - exp(logvar))) as fp32 tensors; the KL term is a
    0-dim tensor summed in a fixed order."""
    if mu.shape != logvar.shape or mu.shape != eps.shape:
        raise ValueError(f"mu {tuple(mu.shape)}, logvar {tuple(logvar.shape)} and eps {tuple(eps.shape)} must match")
    lib = _lib.require_device()
    mu, logvar, eps = (t.contiguous().float() for t in (mu, logvar, eps))
    z = torch.empty_like(mu)
    kld = torch.empty((), dtype=torch.float32, device=mu.device)
    check(lib.b200_vae_reparam_kld(mu.data_ptr(), logvar.data_ptr(), eps.data_ptr(), z.data_ptr(), kld.data_ptr(),
                                   mu.numel(), _stream()), "b200_vae_reparam_kld")
    return z, kld


def avgpool2(x: CL) -> CL:
    """nn.AvgPool{2,3}d(2, 2): floor extents; a 2-D tensor keeps its D slices."""
    sd = x.spatial_dims
    dims = (x.D // 2 if sd == 3 else x.D, x.H // 2, x.W // 2)
    return _resample(x, dims, _lib.INTERPOLATE_AREA, src=(dims[0] * 2 if sd == 3 else x.D, dims[1] * 2, dims[2] * 2))


def _resample(x: CL, dims: Sequence[int], mode: int, src: Sequence[int] | None = None,
              y: torch.Tensor | None = None) -> CL:
    """One b200_interpolate launch (``mode`` B200_INTERPOLATE_NEAREST or _AREA) from x's first ``src`` voxels per axis
    (all of them by default) to extents ``dims``, into ``y`` ([N, *dims, pitch] of x's storage type; a new tensor by
    default).  All three axes are resampled, so a 2-D tensor's D slices are kept as they are, and all ``pitch``
    channels, so the output's pad channels come from the input's (zeros stay zeros).  The ratios are fp32(in / out)
    per axis, interpolate_plan's rule for a size.  AREA over even extents halved is AvgPool(2, 2)."""
    lib = _lib.require_device()
    t = x.t
    N_, D, H, W, P = t.shape
    OD, OH, OW = dims
    if src is not None:
        D, H, W = src
    if y is None:
        y = torch.empty((N_, OD, OH, OW, P), dtype=t.dtype, device=t.device)
    xs, ys = t.stride(), y.stride()
    # the ratios are rounded to fp32 by the c_float arguments
    check(lib.b200_interpolate(t.data_ptr(), DT_H16, (C.c_int64 * 5)(xs[0], 1, xs[1], xs[2], xs[3]), y.data_ptr(),
                               DT_H16, (C.c_int64 * 5)(ys[0], 1, ys[1], ys[2], ys[3]), N_, P, D, H, W, OD, OH, OW, 3,
                               mode, D / OD, H / OH, W / OW, _stream()), "b200_interpolate")
    return CL(y, x.C, x.spatial_dims)


_POOL_MODES = {"avg": _lib.POOL_AVG, "max": _lib.POOL_MAX}


def pool_s2(x: CL, kernel: int, padding: int, mode: str) -> CL:
    """nn.AvgPool{2,3}d (count_include_pad=True) / nn.MaxPool{2,3}d with the given kernel, stride 2 and padding."""
    if mode not in _POOL_MODES:
        raise ValueError(f"unknown pooling mode {mode!r}; expected one of {sorted(_POOL_MODES)}")
    lib = _lib.require_device()
    sd = x.spatial_dims
    o = lambda i: (i + 2 * padding - kernel) // 2 + 1
    dims = (o(x.D) if sd == 3 else x.D, o(x.H), o(x.W))
    if min(dims) < 1 or 2 * padding > kernel:
        raise ValueError(f"pooling kernel {kernel} / padding {padding} does not fit input {(x.D, x.H, x.W)}")
    out = x.like(dims=dims)
    check(lib.b200_pool_s2(x.t.data_ptr(), x.N, x.D, x.H, x.W, x.pitch, sd, kernel, padding, _POOL_MODES[mode],
                           out.t.data_ptr(), _stream()), "b200_pool_s2")
    return out


# F.interpolate mode -> (b200_interpolate mode, the numbers of spatial dims it takes)
_INTERPOLATE_MODES = {"nearest": (_lib.INTERPOLATE_NEAREST, (1, 2, 3)), "linear": (_lib.INTERPOLATE_LINEAR, (1,)),
                      "bilinear": (_lib.INTERPOLATE_BILINEAR, (2,)), "bicubic": (_lib.INTERPOLATE_BICUBIC, (2,)),
                      "trilinear": (_lib.INTERPOLATE_TRILINEAR, (3,)), "area": (_lib.INTERPOLATE_AREA, (1, 2, 3))}


def _f32(v: float) -> float:
    """v rounded to the nearest fp32 value (C's static_cast<float> of a double)."""
    return struct.unpack("f", struct.pack("f", v))[0]


def interpolate_plan(in_sizes: Sequence[int], size=None, scale_factor=None,
                     mode: str = "nearest") -> tuple[list[int], list[float]]:
    """F.interpolate's argument rules (align_corners=False, antialias=False, recompute_scale_factor=None) for an input
    with spatial extents ``in_sizes``: the output extents and the per-axis fp32 ratios b200_interpolate takes.

    Raises what F.interpolate raises for the same arguments, in the same order: ``ValueError`` for both or neither of
    size / scale_factor and for a sequence of the wrong length, ``TypeError`` for a non-integer size, then
    ``NotImplementedError`` for a mode the input's rank does not take.  With a scale factor s the output extent is
    int(in * s) in double precision (ATen's compute_output_size) and the ratio float(1.0 / s); with a size the ratio is
    float(in) / out (ATen's compute_scales_value).  With an odd extent the two differ: 17 -> 8 is ratio 2 with
    scale_factor=0.5 but 2.125 with size=8."""
    dim = len(in_sizes)
    if size is not None and scale_factor is not None:
        raise ValueError("only one of size or scale_factor should be defined")
    if size is not None:
        sizes = list(size) if isinstance(size, (list, tuple)) else [size] * dim
        if len(sizes) != dim:
            raise ValueError(f"Input and output must have the same number of spatial dimensions, but got input "
                             f"with spatial dimensions of {list(in_sizes)} and output size of {size}.")
        if not all(isinstance(v, numbers.Integral) or (torch.is_tensor(v) and not v.is_floating_point()) for v in sizes):
            raise TypeError(f"expected size to be one of int or Tuple[int] or Tuple[int, int] or Tuple[int, int, "
                            f"int], but got size with types {[type(v) for v in sizes]}")
        out = [int(v) for v in sizes]
        scales = [None] * dim
    elif scale_factor is not None:
        if isinstance(scale_factor, (list, tuple)):
            if len(scale_factor) != dim:
                raise ValueError(f"Input and scale_factor must have the same number of spatial dimensions, but got "
                                 f"input with spatial dimensions of {list(in_sizes)} and scale_factor of shape "
                                 f"{scale_factor}.")
            scales = [float(s) for s in scale_factor]
        else:
            scales = [float(scale_factor)] * dim
        out = [int(i * s) for i, s in zip(in_sizes, scales)]
    else:
        raise ValueError("either size or scale_factor should be defined")
    if mode not in _INTERPOLATE_MODES or dim not in _INTERPOLATE_MODES[mode][1]:
        if 1 <= dim <= 3 and mode in ("linear", "bilinear", "trilinear"):
            need = {"linear": 3, "bilinear": 4, "trilinear": 5}[mode]
            raise NotImplementedError(f"Got {dim + 2}D input, but {mode} mode needs {need}D input")
        raise NotImplementedError(f"Input Error: Only 3D, 4D and 5D input Tensors supported (got {dim + 2}D) for the "
                                  f"modes: nearest | linear | bilinear | bicubic | trilinear | area | nearest-exact (got {mode})")
    if min(out) < 1:
        raise RuntimeError(f"Input and output sizes should be greater than 0, but got input {list(in_sizes)} and "
                           f"output {out}")
    ratios = [_f32(1.0 / s) if s is not None and s > 0 else _f32(float(i) / o) for i, o, s in zip(in_sizes, out, scales)]
    return out, ratios


def interpolate(x: torch.Tensor | CL, size=None, scale_factor=None, mode: str = "nearest", *,
                planar_out: bool = False) -> torch.Tensor | CL:
    """F.interpolate(x, size=... | scale_factor=..., mode=mode, align_corners=False) in one b200_interpolate launch.

    ``x`` is either a planar fp32 NC[D]HW tensor (3-, 4- or 5-D, any strides), giving a planar fp32 tensor, or a
    :class:`CL` whose storage ``t`` is h16 or fp32 (``spatial_dims`` 1, 2 or 3; a 1-D CL has D == H == 1), giving a
    CL of the same storage type and pitch, or with ``planar_out`` an NC[D]HW fp32 tensor.  Argument rules and
    exceptions: :func:`interpolate_plan`."""
    dts = {H16: DT_H16, torch.float32: DT_F32}
    cl = isinstance(x, CL)
    t = x.t if cl else x
    sd = x.spatial_dims if cl else x.dim() - 2
    in_sizes = (x.D, x.H, x.W)[3 - sd:] if cl else tuple(x.shape[2:])
    out_sizes, ratios = interpolate_plan(in_sizes, size, scale_factor, mode)
    if t.dtype not in (dts if cl else (torch.float32,)):
        raise TypeError(f"interpolate reads fp32 planar or h16 / fp32 channels-last tensors, got {t.dtype}")
    if cl:
        N, C_ = x.N, x.C
        x_strides = (t.stride(0), 1, t.stride(1), t.stride(2), t.stride(3))
    else:
        N, C_ = x.shape[:2]
        s = x.stride()
        x_strides = (s[0], s[1], *(0,) * (3 - sd), *s[2:])
    lib = _lib.require_device()
    pad = (1,) * (3 - sd)
    if cl and not planar_out:
        y = torch.empty((N, *pad, *out_sizes, x.pitch), dtype=t.dtype, device=t.device)
        res = CL(y, C_, sd)
        y_strides, y_dt = (y.stride(0), 1, y.stride(1), y.stride(2), y.stride(3)), dts[t.dtype]
    else:
        y = res = torch.empty((N, C_, *out_sizes), dtype=torch.float32, device=t.device)
        s = y.stride()
        y_strides, y_dt = (s[0], s[1], *(0,) * (3 - sd), *s[2:]), DT_F32
    r = [1.0] * (3 - sd) + ratios
    check(lib.b200_interpolate(t.data_ptr(), dts[t.dtype], (C.c_int64 * 5)(*x_strides), y.data_ptr(), y_dt,
                               (C.c_int64 * 5)(*y_strides), N, C_, *pad, *in_sizes, *pad, *out_sizes, sd,
                               _INTERPOLATE_MODES[mode][0], *r, _stream()), "b200_interpolate")
    return res


def batchnorm_fold(weight: torch.Tensor, bias: torch.Tensor | None, gamma: torch.Tensor, beta: torch.Tensor,
                   mean: torch.Tensor, var: torch.Tensor, eps: float) -> tuple[torch.Tensor, torch.Tensor]:
    """(w * s, beta + (b - mean) * s) with s = gamma / sqrt(var + eps) per output channel: an eval-mode BatchNorm folded
    into the convolution before it, as fp32 tensors ready for PackedConv."""
    lib = _lib.require_device()
    w = _src_f32(weight)
    b, g, bt, m, v = (None if t is None else _src_f32(t) for t in (bias, gamma, beta, mean, var))
    cout = w.shape[0]
    if any(t.numel() != cout for t in (g, bt, m, v)) or (b is not None and b.numel() != cout):
        raise ValueError(f"BatchNorm parameters do not match the convolution's {cout} output channels")
    w_out = torch.empty_like(w)
    b_out = torch.empty(cout, dtype=torch.float32, device=w.device)
    check(lib.b200_batchnorm_fold(w.data_ptr(), _ptr(b), g.data_ptr(), bt.data_ptr(), m.data_ptr(), v.data_ptr(), eps,
                                  cout, w.numel() // cout, w_out.data_ptr(), b_out.data_ptr(), _stream()),
          "b200_batchnorm_fold")
    return w_out, b_out


def axpy(a: CL, b: CL, alpha: float = 1.0, inplace: bool = False) -> CL:
    """a + alpha * b (same shape)."""
    lib = _lib.require_device()
    if a.t.shape != b.t.shape:
        raise ValueError(f"axpy shape mismatch {tuple(a.t.shape)} vs {tuple(b.t.shape)}")
    out = a if inplace else a.like()
    out.gn = None
    check(lib.b200_axpy_h16(a.t.data_ptr(), b.t.data_ptr(), alpha, out.t.data_ptr(), a.t.numel(), _stream()),
          "b200_axpy_h16")
    return out


def concat(srcs: Sequence[CL]) -> CL:
    """Materialised channel concat (only used where an identity skip needs the raw concatenated tensor)."""
    lib = _lib.require_device()
    a0 = srcs[0]
    out = a0.like(sum(a.C for a in srcs))
    rows = a0.N * a0.spatial
    off = 0
    for a in srcs:
        check(lib.b200_copy_channels(a.t.data_ptr(), a.C, a.pitch, out.t.data_ptr(), out.pitch, off, rows, _stream()),
              "b200_copy_channels")
        off += a.C
    if out.pitch > off:
        out.t[..., off:].zero_()
    return out


def add_f32(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a + b for small fp32 tensors (time + class embedding), via the fused linear-combination kernel."""
    lib = _lib.require_device()
    a = a.contiguous().float()
    b = b.contiguous().float()
    out = torch.empty_like(a)
    c = PndmCoef()
    c.w[0], c.w[1], c.n_hist = 1.0, 1.0, 2
    hist = (C.c_void_p * 2)(a.data_ptr(), b.data_ptr())
    check(lib.b200_pndm_step(hist, None, C.byref(c), None, out.data_ptr(), a.numel(), _stream()), "b200_pndm_step")
    return out


def exp_half_clamped(x: torch.Tensor, lo: float, hi: float) -> torch.Tensor:
    lib = _lib.require_device()
    x = x.contiguous().float()
    y = torch.empty_like(x)
    check(lib.b200_exp_half_clamped(x.data_ptr(), lo, hi, y.data_ptr(), x.numel(), _stream()), "b200_exp_half_clamped")
    return y


def scale_f32(x: torch.Tensor, mul: float = 1.0, divide_by: float | None = None) -> torch.Tensor:
    """x * mul, or x / divide_by when ``divide_by`` is given (exact division, like the reference's ``latent / s``)."""
    if divide_by is not None:
        mul, div = 1.0, float(divide_by)
    else:
        div = 1.0
    if mul == 1.0 and div == 1.0:
        return x
    lib = _lib.require_device()
    x32 = x.contiguous().float()
    y = torch.empty_like(x32)
    check(lib.b200_scale_f32(x32.data_ptr(), float(mul), div, y.data_ptr(), x32.numel(), _stream()), "b200_scale_f32")
    return y if x.dtype == torch.float32 else y.to(x.dtype)


def fma_f32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
    lib = _lib.require_device()
    a, b, c = (t.contiguous().float() for t in (a, b, c))
    y = torch.empty_like(a)
    check(lib.b200_fma_f32(a.data_ptr(), b.data_ptr(), c.data_ptr(), y.data_ptr(), a.numel(), _stream()), "b200_fma_f32")
    return y


def geglu(x: CL) -> CL:
    lib = _lib.require_device()
    Hh = x.C // 2
    out = x.like(Hh)
    M = x.N * x.spatial
    check(lib.b200_geglu(x.t.data_ptr(), M, Hh, x.pitch, out.t.data_ptr(), out.pitch, _stream()), "b200_geglu")
    return out


def linear_geglu(x: CL, pl: PackedLinear) -> CL:
    """a * gelu(gate) with (a, gate) = chunk(x @ W^T + b, 2): linear1 and the gating of a GEGLU feed-forward as ONE
    GEMM (``pl`` from :meth:`PackedLinear.geglu`); the 2H-wide intermediate never exists."""
    H = getattr(pl, "geglu_hidden", None)
    if H is None:
        raise ValueError("linear_geglu needs a PackedLinear.geglu weight")
    if x.C != pl.K:
        raise ValueError(f"linear expects {pl.K} input features, got {x.C}")
    out = x.like(H)
    p = _conv_params([x], pl.w, pl.segs, (1, 1, 1), out.t, (x.D, x.H, x.W), pl.cout, DT_H16, pl.bias, None, ACT_GEGLU,
                     1.0, None, DT_H16, ACT_NONE)
    p.out_cols = out.pitch          # H (a multiple of 32) channels are stored per row, not the GEMM's 2H columns
    igemm_raw(p)
    return out


# --------------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------------
_TC_ATTN_MIN_S = 64
_FLASH_HEAD_DIMS = (64, 128, 256, 512)
_FORCE_UNFUSED_ATTENTION = False      # tests flip this to cover the GEMM + softmax + GEMM path
_ATTN_CHUNK_BYTES = 6 << 30   # fp32 score slab per query chunk


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, dh: int, scale: float,
              vt: torch.Tensor | None = None, residual: torch.Tensor | None = None) -> torch.Tensor:
    """softmax(scale * Q K^T) V on packed [B, T, pitch] h16 rows (heads are channel slices).

    Tensor-core paths (head_dim % 64 == 0, S >= 64; ``vt`` must hold V^T ``[B, H*dh, S_pitch]``, produced for free
    by swapping the operands of the V projection):
      * head_dim in {64, 128, 256, 512}: the flash-style wgmma kernel — scores stay in registers, online softmax;
      * other multiples of 64 (e.g. 768): per (batch, head) QK^T -> fp32 scores (+ softmax partials from the GEMM
        epilogue), one-pass row softmax -> h16, PV, in query slabs so the score matrix never exceeds a few GB.
    Everything else runs on the CUDA-core online-softmax kernel.  ``residual`` ([B, T, pitch] h16) is added in
    the PV epilogue on the tensor-core path only (callers add it themselves otherwise).
    """
    lib = _lib.require_device()
    B, T, _ = q.shape
    S = k.shape[1]
    # row pitches come from the strides: q and k may be column slices of ONE fused [B, T, 2C] projection
    qp, kp = q.stride(1), k.stride(1)
    for name, t_ in (("q", q), ("k", k)):
        if (t_.stride(2) != 1 or (B > 1 and t_.stride(0) != t_.shape[1] * t_.stride(1)) or t_.stride(1) % 8
                or t_.data_ptr() % 16):
            raise ValueError(f"attention: {name} must be rows of a packed [B, T, pitch] tensor (pitch % 8 == 0)")
    out = torch.empty((B, T, round_up(heads * dh, 8)), dtype=H16, device=q.device)
    use_tc = (dh % 64 == 0) and S >= _TC_ATTN_MIN_S and vt is not None
    if not use_tc:
        if residual is not None:
            raise ValueError("residual fusion is only available on the tensor-core attention path")
        if out.shape[2] > heads * dh:
            out.zero_()
        check(lib.b200_attention_small(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, T, S, heads, dh,
                                       qp, kp, v.shape[2], out.shape[2], scale, _stream()),
              "b200_attention_small")
        return out
    if dh in _FLASH_HEAD_DIMS and not _FORCE_UNFUSED_ATTENTION:
        fp = _lib.FlashParams()
        fp.q, fp.k, fp.vt, fp.out = q.data_ptr(), k.data_ptr(), vt.data_ptr(), out.data_ptr()
        fp.res = _ptr(residual)
        fp.B, fp.T, fp.S, fp.heads, fp.dh = B, T, S, heads, dh
        fp.q_pitch, fp.k_pitch, fp.vt_pitch, fp.out_pitch = qp, kp, vt.shape[2], out.shape[2]
        fp.res_pitch = 0 if residual is None else residual.shape[2]
        fp.scale = scale
        if out.shape[2] > heads * dh:
            out.zero_()
        check(lib.b200_attention_flash(C.byref(fp), _stream()), "b200_attention_flash")
        return out
    Sp = round_up(S, 8)
    chunk = max(128, min(T, (_ATTN_CHUNK_BYTES // (4 * Sp)) // 128 * 128))
    scores = torch.empty((min(chunk, T), Sp), dtype=torch.float32, device=q.device)
    probs = torch.empty((min(chunk, T), Sp), dtype=H16, device=q.device)
    n_tiles = (Sp + 127) // 128
    partials = torch.empty((min(chunk, T), n_tiles, 2), dtype=torch.float32, device=q.device)
    nk = round_up(dh, 64) // 64
    ns = round_up(S, 64) // 64
    for b in range(B):
        for h in range(heads):
            for t0 in range(0, T, chunk):
                tc = min(chunk, T - t0)
                # scores = scale * Q_h K_h^T   (A = Q rows, "weights" = K rows, both K-major over dh)
                p = IgemmParams()
                p.a_ptr[0] = q.data_ptr() + ((b * T + t0) * qp + h * dh) * 2
                p.a_C[0], p.a_pitch[0] = dh, qp
                p.in_N, p.in_D, p.in_H, p.in_W = 1, 1, 1, tc
                p.stride_d = p.stride_h = p.stride_w = 1
                p.w_ptr = k.data_ptr() + (b * S * kp + h * dh) * 2
                p.w_rows, p.w_pitch, p.w_K = S, kp, dh
                _fill_segs(p, [(0, 0, 0, 0, 0, nk)])
                p.out_ptr, p.out_dtype = scores.data_ptr(), DT_F32
                p.out_N, p.out_D, p.out_H, p.out_W = 1, 1, 1, tc
                p.cout, p.out_cols = S, Sp
                p.out_sN, p.out_sD, p.out_sH, p.out_sW = tc * Sp, tc * Sp, tc * Sp, Sp
                p.act1, p.scale, p.act2 = ACT_NONE, scale, ACT_NONE
                p.stat_ptr = partials.data_ptr()     # epilogue leaves (max, sum exp) per 128-column tile
                igemm_raw(p)
                check(lib.b200_softmax_rows_partials(scores.data_ptr(), tc, S, Sp, partials.data_ptr(), n_tiles,
                                                     probs.data_ptr(), Sp, _stream()), "b200_softmax_rows_partials")
                # out = P V   (A = P rows over S, "weights" = V^T rows over S)
                p2 = IgemmParams()
                p2.a_ptr[0] = probs.data_ptr()
                p2.a_C[0], p2.a_pitch[0] = S, Sp
                p2.in_N, p2.in_D, p2.in_H, p2.in_W = 1, 1, 1, tc
                p2.stride_d = p2.stride_h = p2.stride_w = 1
                vtp = vt.shape[2]
                p2.w_ptr = vt.data_ptr() + ((b * heads * dh + h * dh) * vtp) * 2
                p2.w_rows, p2.w_pitch, p2.w_K = dh, vtp, S
                _fill_segs(p2, [(0, 0, 0, 0, 0, ns)])
                op = out.shape[2]
                p2.out_ptr, p2.out_dtype = out.data_ptr() + ((b * T + t0) * op + h * dh) * 2, DT_H16
                p2.out_N, p2.out_D, p2.out_H, p2.out_W = 1, 1, 1, tc
                p2.cout, p2.out_cols = dh, dh
                p2.out_sN, p2.out_sD, p2.out_sH, p2.out_sW = tc * op, tc * op, tc * op, op
                p2.act1, p2.scale, p2.act2 = ACT_NONE, 1.0, ACT_NONE
                if residual is not None:
                    rp = residual.shape[2]
                    p2.res_ptr, p2.res_dtype = residual.data_ptr() + ((b * T + t0) * rp + h * dh) * 2, DT_H16
                    p2.res_sN, p2.res_sD, p2.res_sH, p2.res_sW = tc * rp, tc * rp, tc * rp, rp
                igemm_raw(p2)
    return out


def linear_transposed_out(x: torch.Tensor, pl: PackedLinear) -> torch.Tensor:
    """The output buffer of :func:`linear_transposed` (allocate it on the main stream before an ops.fork())."""
    B, S, _ = x.shape
    Sp = round_up(S, 8)
    out = torch.empty((B, pl.cout, Sp), dtype=H16, device=x.device)
    if Sp > S:
        out.zero_()
    return out


def linear_transposed(x: torch.Tensor, C_in: int, pl: PackedLinear, out: torch.Tensor | None = None) -> torch.Tensor:
    """V^T = W x^T + b:  x is [B, S, pitch] h16 rows; returns [B, O, round_up(S, 8)] h16.

    The projection weight plays the A operand (rows = output features) and the activations play the K-major
    "weight" operand, so the transposed value matrix costs no extra pass.
    """
    B, S, xp = x.shape
    O = pl.cout
    Sp = round_up(S, 8)
    if out is None:
        out = linear_transposed_out(x, pl)
    elif tuple(out.shape) != (B, O, Sp):
        raise ValueError("preallocated V^T output has the wrong shape")
    nk = round_up(C_in, 64) // 64
    # ONE launch for the whole batch: the shared projection matrix is the broadcast A operand, sample b's activations
    # are weight batch b, sample b's V^T is output slice b (a per-sample loop was 352 of the 420 GEMM launches of a
    # C2 forward at batch 32)
    p = IgemmParams()
    p.a_ptr[0] = pl.w.data_ptr()
    p.a_C[0], p.a_pitch[0] = C_in, pl.w.shape[1]
    p.a_broadcast = 1
    p.in_N, p.in_D, p.in_H, p.in_W = B, 1, 1, O
    p.stride_d = p.stride_h = p.stride_w = 1
    p.w_ptr = x.data_ptr()
    p.w_rows, p.w_pitch, p.w_K = S, xp, C_in
    p.w_batched, p.w_bstride = 1, S * xp
    _fill_segs(p, [(0, 0, 0, 0, 0, nk)])
    p.out_ptr, p.out_dtype = out.data_ptr(), DT_H16
    p.out_N, p.out_D, p.out_H, p.out_W = B, 1, 1, O
    p.cout, p.out_cols = S, Sp
    p.out_sN, p.out_sD, p.out_sH, p.out_sW = O * Sp, O * Sp, O * Sp, Sp
    p.act1, p.scale, p.act2 = ACT_NONE, 1.0, ACT_NONE
    p.row_bias = _ptr(pl.bias)       # the linear's bias is per output ROW in this orientation
    igemm_raw(p)
    return out


# --------------------------------------------------------------------------------------------------
# time embedding
# --------------------------------------------------------------------------------------------------
def linear_into_cache(x: CL, B: int, T: int, pl: PackedLinear, cache: torch.Tensor, pos0: int) -> None:
    """cache[b, pos0 + t, :] = x[b * T + t, :] @ W^T (+ b): the K / V projection of T new tokens per sequence written
    straight into a [B, max_seq, pitch] key/value cache by the GEMM epilogue (strided output rows), no copy."""
    if x.C != pl.K:
        raise ValueError(f"linear expects {pl.K} input features, got {x.C}")
    Bc, L, P = cache.shape
    if Bc != B or pos0 + T > L or P != round_up(pl.cout, 8):
        raise ValueError("key/value cache does not match the projection")
    xin = CL(x.t.reshape(B, 1, 1, T, x.pitch), x.C, 2)
    p = _conv_params([xin], pl.w, pl.segs, (1, 1, 1), cache, (1, 1, T), pl.cout, DT_H16, pl.bias, None, ACT_NONE, 1.0,
                     None, DT_H16, ACT_NONE, out_elem_off=pos0 * P, out_strides=(L * P, 0, 0, P))
    igemm_raw(p)


def attention_causal(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, dh: int, scale: float, S: int,
                     causal: bool = True, q_pos0: int = 0, pos_dev: torch.Tensor | None = None) -> torch.Tensor:
    """softmax(scale * Q K^T [+ causal mask]) V for the autoregressive transformer: q [B, T, pitch]; k, v
    [B, rows >= S, pitch] — typically a key/value cache of which the first S rows are valid; query row t sits at
    absolute position q_pos0 + t and, if causal, sees keys <= its position (blocks/selfattention.py:121-140)."""
    lib = _lib.require_device()
    B, T, qp = q.shape
    out = torch.empty((B, T, round_up(heads * dh, 8)), dtype=H16, device=q.device)
    if out.shape[2] > heads * dh:
        out.zero_()
    check(lib.b200_attention_small_ex(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, T, S, heads, dh, qp,
                                      k.shape[2], v.shape[2], out.shape[2], scale, k.shape[1], int(causal), q_pos0,
                                      _ptr(pos_dev), _stream()), "b200_attention_small_ex")
    return out


def rows_linear(x: torch.Tensor, K: int, pl: PackedLinear, *, ln=None, act: int = ACT_NONE,
                residual: torch.Tensor | None = None, out_f32: bool = False) -> torch.Tensor:
    """Decode-time linear layer on M <= 8 h16 rows ``x`` [M, pitch]: act(LN?(x) @ W^T + b) + residual, one GEMV
    kernel (b200_rows_linear).  ``ln`` = (gamma, beta, eps) fuses the preceding LayerNorm."""
    lib = _lib.require_device()
    M = x.shape[0]
    if K != pl.K:
        raise ValueError(f"linear expects {pl.K} input features, got {K}")
    out = torch.empty((M, round_up(pl.cout, 4 if out_f32 else 8)), dtype=torch.float32 if out_f32 else H16,
                      device=x.device)
    if out.shape[1] > pl.cout:
        out.zero_()
    g, b, eps = (ln[0].data_ptr(), ln[1].data_ptr(), float(ln[2])) if ln is not None else (None, None, 0.0)
    check(lib.b200_rows_linear(x.data_ptr(), x.shape[1], M, K, g, b, eps, pl.w.data_ptr(), pl.w.shape[1], pl.cout,
                               _ptr(pl.bias), act, _ptr(residual), 0 if residual is None else residual.shape[1],
                               out.data_ptr(), out.shape[1], DT_F32 if out_f32 else DT_H16, _stream()),
          "b200_rows_linear")
    return out


def attention_decode(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, dh: int, scale: float, S: int,
                     pos_dev: torch.Tensor | None = None) -> torch.Tensor:
    """One query row per sequence ([B, pitch]) over the first S rows of the key / value caches [B, rows, pitch]
    (S = *pos_dev + 1 when ``pos_dev`` is given)."""
    lib = _lib.require_device()
    B = q.shape[0]
    out = torch.empty((B, round_up(heads * dh, 8)), dtype=H16, device=q.device)
    if out.shape[1] > heads * dh:
        out.zero_()
    check(lib.b200_attention_decode(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, S, heads, dh,
                                    q.shape[1], k.shape[2], v.shape[2], out.shape[1], scale, k.shape[1], _ptr(pos_dev),
                                    _stream()), "b200_attention_decode")
    return out


def cache_append(src: torch.Tensor, cache: torch.Tensor, T: int, pos_dev: torch.Tensor) -> None:
    """cache[b, *pos_dev + t, :] = src[b * T + t, :] with the position read on the device (graph-captured decoding)."""
    lib = _lib.require_device()
    B, L, P = cache.shape
    check(lib.b200_cache_append(src.data_ptr(), cache.data_ptr(), B, T, L, P, pos_dev.data_ptr(), _stream()),
          "b200_cache_append")


def advance_i32(p: torch.Tensor, delta: int) -> None:
    check(_lib.require_device().b200_advance_i32(p.data_ptr(), delta, _stream()), "b200_advance_i32")


def embed_tokens(tokens: torch.Tensor, tok_emb: torch.Tensor, pos_emb: torch.Tensor, pos0: int = 0,
                 pos_dev: torch.Tensor | None = None) -> CL:
    """Token + absolute-position embedding rows of an int64 [B, T] index tensor -> CL rows [1, 1, 1, B*T, pitch]."""
    lib = _lib.require_device()
    B, T = tokens.shape
    C_ = tok_emb.shape[1]
    tk = tokens if (tokens.dtype == torch.int64 and tokens.is_contiguous()) else tokens.long().contiguous()
    out = torch.empty((1, 1, 1, B * T, round_up(C_, 8)), dtype=H16, device=tokens.device)
    check(lib.b200_embed_tokens(tk.data_ptr(), B * T, T, pos0, tok_emb.data_ptr(), pos_emb.data_ptr(), C_,
                                out.data_ptr(), out.shape[-1], _ptr(pos_dev), _stream()), "b200_embed_tokens")
    return CL(out, C_, 2)


def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    lib = _lib.require_device()
    t = t.contiguous().float()
    emb = torch.empty((t.shape[0], dim), dtype=torch.float32, device=t.device)
    check(lib.b200_timestep_embedding(t.data_ptr(), t.shape[0], dim, max_period, emb.data_ptr(), _stream()),
          "b200_timestep_embedding")
    return emb


def small_linear(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor | None, act_in: int = ACT_NONE,
                 act_out: int = ACT_NONE) -> torch.Tensor:
    """fp32 GEMV-class linear for the time-embedding path (M = batch rows)."""
    lib = _lib.require_device()
    x = x.contiguous().float()
    M, K = x.shape
    O = weight.shape[0]
    y = torch.empty((M, O), dtype=torch.float32, device=x.device)
    w = weight if weight.dtype == torch.float32 and weight.is_contiguous() else weight.detach().float().contiguous()
    b = None if bias is None else (bias if bias.dtype == torch.float32 else bias.detach().float())
    check(lib.b200_small_linear(x.data_ptr(), M, K, w.data_ptr(), _ptr(b), O, act_in, act_out, y.data_ptr(), _stream()),
          "b200_small_linear")
    return y


# ------------------------------------------------------------------------------------------------
# Sample-quality metrics (generativemodels_b200.metrics).  Inputs are planar [N, C, D, H, W] views of any strides in
# fp32 / fp64 / fp16 / bf16, read in place; everything the kernels compute is fp32 with fp64 sums.
# ------------------------------------------------------------------------------------------------
_METRIC_DT = {torch.float32: _lib.DT_F32, torch.float64: _lib.DT_F64, torch.float16: _lib.DT_FP16,
              torch.bfloat16: _lib.DT_BF16}


def _metric_dt(t: torch.Tensor) -> int:
    if t.dtype not in _METRIC_DT:
        raise TypeError(f"metrics read fp32, fp64, fp16 or bf16 tensors, got {t.dtype}")
    return _METRIC_DT[t.dtype]


@dataclass
class SsimScale:
    """What one b200_ssim pass leaves for b200_ssim_combine: per-CTA fp64 sums [N, slots, 2] and the voxel count per
    item (C * OD * OH * OW) that turns them into means."""
    partials: torch.Tensor
    slots: int
    count: int


def ssim_pass(x: torch.Tensor, y: torch.Tensor, taps: Sequence[Sequence[float]], scale: float, c1: float, c2: float,
              maps: bool = False) -> tuple[SsimScale, torch.Tensor | None, torch.Tensor | None]:
    """One fused SSIM / CS pass over 5-D [N, C, D, H, W] views x (= y_pred) and y with the separable kernel
    ``taps = (taps_d, taps_h, taps_w)``; with ``maps`` also the fp32 SSIM and CS maps [N, C, OD, OH, OW]."""
    lib = _lib.require_device()
    p = _lib.SsimParams()
    p.x, p.y = x.data_ptr(), y.data_ptr()
    p.x_dtype, p.y_dtype = _metric_dt(x), _metric_dt(y)
    p.x_strides[:], p.y_strides[:] = x.stride(), y.stride()
    p.N, p.C, p.D, p.H, p.W = x.shape
    p.kd, p.kh, p.kw = (len(t) for t in taps)
    if max(p.kd, p.kh, p.kw) > _lib.SSIM_MAX_K:
        raise NotImplementedError(f"SSIM kernels are at most {_lib.SSIM_MAX_K} taps per axis, got {p.kd, p.kh, p.kw}")
    for dst, t in zip((p.taps_d, p.taps_h, p.taps_w), taps):
        dst[:len(t)] = list(t)
    p.scale, p.c1, p.c2 = scale, c1, c2
    nbytes = lib.b200_ssim_workspace_bytes(C.byref(p))
    if nbytes < 0:
        raise NotImplementedError(f"no SSIM kernel for a {p.kd} x {p.kh} x {p.kw} kernel on a {p.D} x {p.H} x {p.W} "
                                  "input (the tile does not fit in shared memory)")
    part = torch.empty(nbytes // 8, dtype=torch.float64, device=x.device)
    out_shape = (p.N, p.C, p.D - p.kd + 1, p.H - p.kh + 1, p.W - p.kw + 1)
    ssim_map = cs_map = None
    if maps:
        ssim_map = torch.empty(out_shape, dtype=torch.float32, device=x.device)
        cs_map = torch.empty(out_shape, dtype=torch.float32, device=x.device)
    p.ssim_map, p.cs_map, p.partials = _ptr(ssim_map), _ptr(cs_map), part.data_ptr()
    check(lib.b200_ssim(C.byref(p), _stream()), "b200_ssim")
    count = out_shape[1] * out_shape[2] * out_shape[3] * out_shape[4]
    return SsimScale(part, nbytes // (16 * p.N), count), ssim_map, cs_map


def ssim_combine(scales: Sequence[SsimScale], N: int, weights: Sequence[float] | None = None):
    """Per-item means of SSIM and CS per scale (fp32 [S, N] each) and, with ``weights`` (one per scale), MS-SSIM
    prod_s relu(v_s) ** w_s (fp32 [N]; v_s = the CS mean, the SSIM mean at the last scale)."""
    lib = _lib.require_device()
    if not 1 <= len(scales) <= _lib.SSIM_MAX_SCALES:
        raise NotImplementedError(f"MS-SSIM takes 1 to {_lib.SSIM_MAX_SCALES} scales, got {len(scales)}")
    dev = scales[0].partials.device
    p = _lib.SsimCombineParams()
    for i, s in enumerate(scales):
        p.partials[i], p.slots[i], p.count[i] = s.partials.data_ptr(), s.slots, s.count
        p.weights[i] = float(weights[i]) if weights is not None else 0.0
    p.N, p.n_scales = N, len(scales)
    ssim = torch.empty((len(scales), N), dtype=torch.float32, device=dev)
    cs = torch.empty((len(scales), N), dtype=torch.float32, device=dev)
    ms = torch.empty(N, dtype=torch.float32, device=dev) if weights is not None else None
    p.ssim_mean, p.cs_mean, p.ms_ssim = ssim.data_ptr(), cs.data_ptr(), _ptr(ms)
    check(lib.b200_ssim_combine(C.byref(p), _stream()), "b200_ssim_combine")
    return ssim, cs, ms


def avgpool2_f32(x: torch.Tensor, dims: int) -> torch.Tensor:
    """F.avg_pool{dims}d(x, kernel_size=2) in fp32 on a 5-D [N, C, D, H, W] view (2-D: D == 1, not pooled); a
    contiguous fp32 result.  b200_interpolate's AREA over the even part of each pooled extent."""
    lib = _lib.require_device()
    N_, C_, D, H, W = x.shape
    y = torch.empty((N_, C_, D // 2 if dims == 3 else D, H // 2, W // 2), dtype=torch.float32, device=x.device)
    src = [2 * v for v in y.shape[2:]]
    if dims == 2:
        src[0] = D
    check(lib.b200_interpolate(x.data_ptr(), _metric_dt(x), (C.c_int64 * 5)(*x.stride()), y.data_ptr(), DT_F32,
                               (C.c_int64 * 5)(*y.stride()), N_, C_, *src, *y.shape[2:], dims,
                               _lib.INTERPOLATE_AREA, 1.0, 1.0, 1.0, _stream()), "b200_interpolate")
    return y


def mmd(y: torch.Tensor, y_pred: torch.Tensor) -> torch.Tensor:
    """mean(Y Y^T) + mean(P P^T) - 2 mean(P Y^T) of MMDMetric's linear kernel over the flattened [B, V] rows, as the
    column reduction sum_v (ybar_v - pbar_v)^2 / V; y and y_pred of equal shape, 1 to 5 dims.  fp32 0-dim result."""
    lib = _lib.require_device()
    if y.dim() > 5:
        y, y_pred = y.reshape(y.shape[0], -1), y_pred.reshape(y_pred.shape[0], -1)
    pad = 5 - y.dim()
    shape = (C.c_int64 * 5)(*y.shape, *(1,) * pad)
    ys = (C.c_int64 * 5)(*y.stride(), *(1,) * pad)
    ps = (C.c_int64 * 5)(*y_pred.stride(), *(1,) * pad)
    ws = torch.empty(lib.b200_mmd_workspace_bytes(shape) // 8, dtype=torch.float64, device=y.device)
    out = torch.empty((), dtype=torch.float32, device=y.device)
    check(lib.b200_mmd(y.data_ptr(), _metric_dt(y), ys, y_pred.data_ptr(), _metric_dt(y_pred), ps, shape,
                       ws.data_ptr(), out.data_ptr(), _stream()), "b200_mmd")
    return out


def fid_moments(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """fp64 column mean [F] and covariance (X - mu)^T (X - mu) / (n - 1) [F, F] of a 2-D [n, F] view (n >= 2) of any
    strides in fp32 / fp64 / fp16 / bf16, read in place."""
    lib = _lib.require_device()
    p = _lib.FidMomentsParams()
    p.x, p.x_dtype = x.data_ptr(), _metric_dt(x)
    p.n, p.F = x.shape
    p.x_strides[:] = x.stride()
    mu = torch.empty(p.F, dtype=torch.float64, device=x.device)
    sigma = torch.empty((p.F, p.F), dtype=torch.float64, device=x.device)
    p.mu, p.sigma = mu.data_ptr(), sigma.data_ptr()
    check(lib.b200_fid_moments(C.byref(p), _stream()), "b200_fid_moments")
    return mu, sigma


def frechet(mu_x: torch.Tensor, sigma_x: torch.Tensor, mu_y: torch.Tensor, sigma_y: torch.Tensor,
            details: bool = False):
    """|mu_x - mu_y|^2 + tr sigma_x + tr sigma_y - 2 tr sqrt(sigma_x sigma_y) from contiguous fp64 mu [F] and symmetric
    PSD sigma [F, F]: a 0-dim fp64 tensor; with ``details`` also the F eigenvalues of M = G^T sigma_x G (ascending, fp64)
    and the rank of sigma_y's pivoted Cholesky factor G (0-dim int32)."""
    lib = _lib.require_device()
    F_ = mu_x.shape[0]
    p = _lib.FrechetParams()
    p.mu_x, p.sigma_x, p.mu_y, p.sigma_y = (t.data_ptr() for t in (mu_x, sigma_x, mu_y, sigma_y))
    p.F = F_
    nbytes = lib.b200_frechet_workspace_bytes(F_)
    if nbytes < 0:
        raise NotImplementedError(f"the Frechet distance takes 1 to {_lib.FID_MAX_F} features, got {F_}")
    ws = torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=mu_x.device)
    out = torch.empty((), dtype=torch.float64, device=mu_x.device)
    eig = torch.empty(F_, dtype=torch.float64, device=mu_x.device) if details else None
    rank = torch.empty((), dtype=torch.int32, device=mu_x.device) if details else None
    p.workspace, p.out, p.eigvals, p.rank = ws.data_ptr(), out.data_ptr(), _ptr(eig), _ptr(rank)
    check(lib.b200_frechet(C.byref(p), _stream()), "b200_frechet")
    return (out, eig, rank) if details else out


# ------------------------------------------------------------------------------------------------
# Perceptual distance (generativemodels_b200.losses): the network's input preparation and the feature distance.
# ------------------------------------------------------------------------------------------------
def perceptual_prep(x: torch.Tensor, y: torch.Tensor, strides: Sequence[Sequence[int]], S: int, OH: int, OW: int,
                    idx: torch.Tensor | None, n_out: int, out: torch.Tensor) -> None:
    """b200_perceptual_prep: ``n_out`` z-scored 3-channel images of x and of y into ``out[:n_out]`` and
    ``out[n_out:]`` (h16 [2 * n_out, 1, OH, OW, 8]).  ``strides`` = the {image, channel, slice, row, column} element
    strides of x and of y; ``idx`` (int64, on the device) picks the source images, None takes 0 .. n_out - 1."""
    lib = _lib.require_device()
    half = n_out * OH * OW * 8 * out.element_size()
    check(lib.b200_perceptual_prep(x.data_ptr(), _metric_dt(x), (C.c_int64 * 5)(*strides[0]), y.data_ptr(),
                                   _metric_dt(y), (C.c_int64 * 5)(*strides[1]), x.shape[1], S, OH, OW, _ptr(idx),
                                   n_out, out.data_ptr(), out.data_ptr() + half, _stream()), "b200_perceptual_prep")


def perceptual_distance(fx: torch.Tensor, fy: torch.Tensor, C_: int, image: torch.Tensor,
                        image32: torch.Tensor | None = None) -> None:
    """b200_perceptual_distance of two channels-last feature maps [B, D, H, W, pitch] (fp32 or h16) into the fp64
    per-image values ``image`` [B] (and their fp32 copy ``image32``)."""
    lib = _lib.require_device()
    B = fx.shape[0]
    HW = fx.shape[1] * fx.shape[2] * fx.shape[3]
    dt = DT_F32 if fx.dtype == torch.float32 else DT_H16
    pixel = torch.empty(B * HW, dtype=torch.float32, device=fx.device)
    check(lib.b200_perceptual_distance(fx.data_ptr(), fy.data_ptr(), dt, B, HW, C_, fx.shape[-1], pixel.data_ptr(),
                                       image.data_ptr(), _ptr(image32), _stream()), "b200_perceptual_distance")


def perceptual_mean(image: torch.Tensor, counts: Sequence[int]) -> tuple[torch.Tensor, torch.Tensor]:
    """b200_perceptual_mean: (fp64 [len(counts) + 1] group means and their sum, fp32 0-dim loss)."""
    lib = _lib.require_device()
    means = torch.empty(len(counts) + 1, dtype=torch.float64, device=image.device)
    loss = torch.empty((), dtype=torch.float32, device=image.device)
    check(lib.b200_perceptual_mean(image.data_ptr(), len(counts), (C.c_int32 * len(counts))(*counts),
                                   means.data_ptr(), loss.data_ptr(), _stream()), "b200_perceptual_mean")
    return means, loss

"""b200_igemm on the GPU against tests/igemm_emulator.py, the float64 reading of include/b200gen.h that the CPU suite
uses for the host plumbing of ops.  Every case fills ONE parameter struct twice through the same function, once with
device and once with host pointers, runs the library on the first and the emulator on the second, and checks:

  values     every element of [0, out_cols) of every output voxel against the emulator (bound below);
  padding    columns [cout, out_cols) are exactly +0;
  footprint  the output allocation is larger than the call's footprint (an extra voxel along every axis, out_sW >
             out_cols where the case allows it) and prefilled with a NaN bit pattern that must survive outside it;
  ignored    A channels [a_C, a_pitch), W columns [w_K, w_pitch) and weight rows between batches hold NaN;
  partials   GroupNorm partials summed over slots equal the float64 (sum, sum of squares) of the kernel's own stored
             output and the emulator's slot; softmax partials equal the max / sum of exp of the kernel's own fp32 row;
  determinism  a second identical call is bit-identical (except the check kernel's atomic GroupNorm partials);
  kernel     b200_igemm_plan's column tile and split factor (256 = the two-CTA wide kernel) are what the case names.

Value bound.  mag = the emulator on |A| and |W| without epilogue (sum |a w| per output).  The fp32 accumulation of
exactly representable 16-bit products in any order is within ~sqrt(K) 2^-24 mag of the float64 sum; the bound allows
    |got - want| <= ulp16(max(|got|, |want|)) + C_LIP |scale| 2^-16 mag + REL (|want| + 1)
where the ulp term (16-bit outputs only) covers the two sides rounding to neighbouring 16-bit values, C_LIP = 1.5 covers
the Lipschitz constants of act1 followed by act2 (GELU 1.13, SiLU 1.1, others <= 1), and REL = 2^-17 covers fp32
rounding of the additive terms and __expf in SiLU / sigmoid.  A dropped 64-channel chunk, a wrong bias column or a
swapped activation is off by O(0.1 .. 1) against a bound of ~1e-3 (fp16), ~1e-2 (bf16) or ~1e-5 (fp32).

Case matrix (predicates from generativemodels_b200/csrc/igemm.cu; BN = column tile of igemm_tc_kernel):

  store path        selected by
  lean              lean_ok: fast_ok && no act / scale / row_bias / gn_partial, h16 out, not GEGLU
  fast              fast_ok: out_vec && !out_staged && !stat_ptr && (no residual || h16 res_vec)
  GEGLU             p.geglu (act1 == B200_ACT_GEGLU), BN >= 64
  general vector    !fast_ok with out_vec: fp32 residual, or stat_ptr
  general scalar    out_vec == 0: out_cols % 8 != 0 (h16) or a misaligned out_ptr
  staged            out_staged: fp32 output with out_sW * 4 > 2048
  wide              wide_fits (impl 3)
  split, 2 kernels  make_plan splits > 1, split_ws -> igemm_split_reduce_kernel
  check             impl 1: igemm_check_kernel (+ gn8_partial_check_kernel)

Each CASES row names its path; the persistence rows have N = 2 or 3 with more tiles than SMs (128-column kernel) or
more units than clusters (wide kernel), so CTAs carry the per-sample row vector and GroupNorm partials across a sample
boundary.
"""
import ctypes as C
import zlib
from dataclasses import dataclass, replace

import numpy as np
import pytest
import torch

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import (ACT_GEGLU, ACT_GELU, ACT_LEAKYRELU, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_SILU,
                                         ACT_TANH, B200_EINVAL, DT_F32, DT_H16, IgemmParams)
from tests import igemm_emulator

pytestmark = pytest.mark.gpu

FP16 = ops.H16 is torch.float16
SENT16, SENT32 = 0x7FFF, 0x7FFFFFFF          # NaN in fp16, bf16 and fp32: "never written"


def cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Case:
    name: str
    path: str
    expect: tuple | None          # (column tile, split factor) from b200_igemm_plan; None for impl 1
    in_dhw: tuple                 # input extent (D, H, W)
    out_dhw: tuple
    srcs: tuple                   # ((a_C, a_pitch), ...)
    segs: tuple                   # ((src, dw, dh, dd, c0, nchunks), ...)
    cout: int
    out_cols: int = 0             # 0: cout (GEGLU: cout / 2)
    N: int = 1
    stride: tuple = (1, 1, 1)     # (sd, sh, sw)
    out_f32: bool = False
    out_pad: int = 0              # out_sW = out_cols + out_pad
    out_off: int = 0              # element offset of out_ptr in its allocation
    w_rows: int = 0               # 0: cout
    w_trim: int = 0               # w_K = w_pitch - w_trim (0: w_K = 0, the whole row)
    w_batched: bool = False
    a_broadcast: bool = False
    bias: bool = True
    rowvec: str | None = None     # "sample" (rowvec_bstride = cout + 8) or "bcast" (rowvec_bstride = 0)
    row_bias: bool = False
    act1: int = ACT_NONE
    scale: float = 1.0
    act2: int = ACT_NONE
    res: str | None = None        # "h16" or "f32"
    res_pad: int = 0              # res_sW = out_cols + res_pad
    res_off: int = 0
    stat: bool = False
    gn: int = 0                   # gn_group: 8 or 4 (0 = no partials)
    impl: int = 2
    split: str | None = None      # "two" (split_ws)
    huge: bool = False            # bias of +-1e5 on two thirds of the columns: outputs past the fp16 range

    @property
    def cols(self):
        return self.out_cols or (self.cout // 2 if self.act1 == ACT_GEGLU else self.cout)


def gemm(name, path, expect, M, K, cout, **kw):
    pitch = (K + 7) // 8 * 8 + 8
    return Case(name, path, expect, (1, 1, M), (1, 1, M), ((K, pitch),), ((0, 0, 0, 0, 0, cdiv(K, 64)),), cout, **kw)


def conv(name, path, expect, N, dhw, cins, cout, k=3, s=1, p=1, **kw):
    """k^3 (D > 1) or k^2 (D == 1) convolution, taps outer, sources inner, every source from channel 0."""
    kd, pd, sd = (k, p, s) if dhw[0] > 1 else (1, 0, 1)
    srcs = tuple((c, (c + 7) // 8 * 8 + 8) for c in cins)
    segs = tuple((i, dw - p, dh - p, dd - pd, 0, cdiv(c, 64))
                 for dd in range(kd) for dh in range(k) for dw in range(k) for i, c in enumerate(cins))
    od = tuple((n + 2 * q - kk) // ss + 1 for n, q, kk, ss in zip(dhw, (pd, p, p), (kd, k, k), (sd, s, s)))
    return Case(name, path, expect, dhw, od, srcs, segs, cout, N=N, stride=(sd, s, s), **kw)


def two_source_c0(name, path, expect, **kw):
    """Stride-2 3x3 over source 0 (100 of 112 channels) and channels 64..191 of source 1 (c0 = 1)."""
    segs = tuple(s for dh in range(3) for dw in range(3) for s in ((0, dw - 1, dh - 1, 0, 0, 2), (1, dw - 1, dh - 1, 0, 1, 2)))
    return Case(name, path, expect, (1, 11, 13), (1, 6, 7), ((100, 112), (192, 200)), segs, 64, stride=(1, 2, 2), **kw)


CASES = [
    # ---- 128-column kernel (impl 2) ----
    gemm("lean_ragged_K", "lean", (64, 1), 300, 300, 64, w_trim=20),
    conv("lean_res256_rowvec_bcast", "lean", (64, 1), 2, (1, 10, 12), [64], 128, res="h16", res_pad=16,
         rowvec="bcast"),
    gemm("lean_res_vec_only_wrows", "lean + general vector tail", (128, 1), 200, 128, 136, out_pad=8, res="h16",
         w_rows=150),
    conv("fast_tanh_scale", "fast", (64, 1), 1, (4, 6, 8), [64], 96, act1=ACT_TANH, scale=0.7, rowvec="sample"),
    conv("fast_relu_sigmoid_res256", "fast", (128, 1), 2, (1, 9, 13), [96], 128, k=1, p=0, act1=ACT_RELU,
         scale=-1.5, act2=ACT_SIGMOID, res="h16", res_pad=32),
    conv("fast_gelu_leaky_stride2", "fast", (64, 1), 2, (1, 17, 15), [64], 64, s=2, act1=ACT_GELU, scale=1.25,
         act2=ACT_LEAKYRELU, rowvec="sample"),
    conv("fast_silu_silu_gn8_two_src", "fast", (64, 1), 2, (1, 12, 10), [64, 32], 64, act1=ACT_SILU, scale=0.5,
         act2=ACT_SILU, gn=8, res="h16", res_pad=8, w_trim=16),
    conv("fast_leaky_tanh_gn4", "fast", (128, 1), 1, (3, 8, 8), [32], 128, k=1, p=0, act1=ACT_LEAKYRELU,
         act2=ACT_TANH, gn=4),
    gemm("fast_sigmoid_gelu_f32", "fast", (128, 1), 257, 192, 128, out_f32=True, out_pad=4, act1=ACT_SIGMOID,
         scale=3.0, act2=ACT_GELU),
    gemm("fast_row_bias_batched_bcast", "fast", (128, 1), 192, 128, 96, N=2, w_batched=True, a_broadcast=True,
         row_bias=True, bias=False),
    gemm("geglu_bn128", "GEGLU", (128, 1), 256, 128, 256, out_pad=16),
    gemm("geglu_bn64_ragged_rows", "GEGLU", (64, 1), 100, 64, 64, out_pad=8),
    conv("general_f32res_vec", "general vector", (64, 1), 2, (1, 8, 12), [64], 64, act1=ACT_SILU, scale=2.0,
         act2=ACT_GELU, res="f32", res_pad=4),
    gemm("general_f32res_scalar_f32out", "general vector", (128, 1), 150, 128, 80, out_f32=True, res="f32", res_off=1,
         act2=ACT_TANH),
    conv("general_scalar_ragged_cols", "general scalar", (64, 1), 1, (1, 7, 9), [64], 67, out_cols=70, w_rows=80,
         act1=ACT_TANH, act2=ACT_SIGMOID, res="h16", res_pad=3),
    gemm("general_scalar_misaligned_out", "general scalar", (64, 1), 130, 256, 64, out_off=1, act1=ACT_LEAKYRELU,
         act2=ACT_RELU, res="h16"),
    gemm("general_stat_res_act2", "general vector + stat", (128, 1), 140, 128, 250, out_cols=392, out_f32=True,
         stat=True, res="f32", res_pad=4, act2=ACT_TANH, scale=0.125),
    gemm("staged_stat", "staged + stat", (128, 1), 96, 64, 600, out_cols=608, out_pad=32, out_f32=True, stat=True,
         scale=0.5),
    conv("staged_conv_f32_res", "staged", (64, 1), 2, (1, 6, 10), [64], 40, out_f32=True, out_pad=480, act1=ACT_GELU,
         res="f32", res_pad=4),
    two_source_c0("two_src_c0_stride2", "fast", (64, 1), act1=ACT_SILU),
    gemm("bn16_pad_cols", "general vector", (16, 1), 160, 64, 10, out_cols=16, act1=ACT_GELU),
    gemm("bn16_lean", "lean", (16, 1), 129, 64, 16),
    conv("bn32_gn8_rowvec", "fast", (32, 1), 2, (1, 8, 8), [64], 32, gn=8, rowvec="sample", act1=ACT_RELU),
    # ---- persistent CTAs across a sample boundary ----
    conv("persist_tc_n3_gn8", "fast", (128, 1), 3, (1, 64, 96), [64], 128, k=1, p=0, rowvec="sample", gn=8,
         act1=ACT_SILU),
    conv("persist_tc_n2_lean_two_col_tiles", "lean", (128, 1), 2, (1, 48, 96), [64], 256, k=1, p=0,
         rowvec="sample", res="h16", res_pad=16),
    conv("persist_tc_n2_gn4_two_col_tiles", "fast", (128, 1), 2, (1, 48, 96), [64], 256, k=1, p=0, rowvec="sample",
         gn=4, scale=0.5),
    conv("persist_wide_n2_gn8", "wide", (256, 1), 2, (1, 96, 96), [64], 256, k=1, p=0, impl=3, rowvec="sample",
         gn=8, act1=ACT_SILU, res="h16", res_pad=16),
    conv("persist_wide_n3_gn4", "wide", (256, 1), 3, (1, 80, 96), [64], 256, k=1, p=0, impl=3, rowvec="sample",
         gn=4),
    # ---- wide kernel ----
    conv("wide_res_vec_tanh_sigmoid", "wide", (256, 1), 2, (4, 6, 10), [64], 256, impl=3, out_pad=8, res="h16",
         res_off=8, act1=ACT_TANH, scale=0.5, act2=ACT_SIGMOID, rowvec="bcast"),
    conv("wide_two_src_gn4_c512", "wide", (256, 1), 1, (1, 12, 20), [64, 96], 512, impl=3, gn=4, act1=ACT_GELU),
    # ---- split reduction (impl 0 with a workspace) ----
    conv("split_two_kernels", "split, 2 kernels", (128, 3), 1, (4, 4, 8), [256], 96, impl=0, split="two",
         act1=ACT_SILU, scale=0.5, act2=ACT_TANH, res="h16", rowvec="sample"),
    conv("split_two_kernels_f32_ragged", "split, 2 kernels", (128, 3), 1, (4, 4, 8), [256], 97, out_cols=100,
         w_rows=112, out_f32=True, impl=0, split="two", act1=ACT_GELU, res="f32", res_pad=4),
    conv("split_two_kernels_n2_misaligned", "split, 2 kernels", (128, 3), 2, (4, 4, 8), [256], 96, impl=0,
         split="two", out_off=1, res="f32", res_off=1, act2=ACT_LEAKYRELU, rowvec="sample"),
    # ---- CUDA-core cross-check kernel ----
    conv("check_gn8_res_gelu_silu", "check", None, 2, (1, 9, 11), [64, 48], 64, out_cols=72, w_rows=70, impl=1, gn=8,
         res="h16", act1=ACT_GELU, act2=ACT_SILU, rowvec="sample"),
    conv("check_f32_scalar_stride2", "check", None, 1, (1, 13, 12), [80], 20, s=2, out_f32=True, out_off=1, impl=1,
         res="f32", res_off=1, act1=ACT_TANH, act2=ACT_SIGMOID),
]

# one case per 16-bit store path, outputs pushed past +-65504 (fp16 stores must saturate, bf16 ones must not)
SATURATION = [
    gemm("sat_lean", "lean", (64, 1), 200, 128, 64, huge=True),
    conv("sat_fast_gn8", "fast", (64, 1), 2, (1, 8, 12), [64], 64, huge=True, act1=ACT_RELU, gn=8),
    gemm("sat_geglu", "GEGLU", (128, 1), 128, 128, 256, huge=True),
    conv("sat_general_vector", "general vector", (64, 1), 2, (1, 8, 12), [64], 64, huge=True, res="f32"),
    gemm("sat_general_scalar", "general scalar", (128, 1), 130, 64, 67, out_cols=70, huge=True),
    conv("sat_split_two", "split, 2 kernels", (128, 3), 1, (4, 4, 8), [256], 96, impl=0, split="two", huge=True),
    conv("sat_wide_gn8", "wide", (256, 1), 1, (4, 6, 10), [64], 256, impl=3, huge=True, gn=8),
    conv("sat_check_gn8", "check", None, 1, (1, 8, 12), [64], 64, impl=1, huge=True, gn=8),
]


# ------------------------------------------------------------------------------------------------------------------
# operands, layout and the one parameter-filling function
# ------------------------------------------------------------------------------------------------------------------
class Geom:
    def __init__(self, c: Case, nsm: int):
        self.OD, self.OH, self.OW = c.out_dhw
        cols = c.cols
        self.sW = cols + c.out_pad
        self.sH = (self.OW + 1) * self.sW             # one extra voxel along every axis: stores past OW / OH / OD land
        self.sD = (self.OH + 1) * self.sH             # on the sentinel
        self.sN = (self.OD + 1) * self.sD
        self.out_len = c.out_off + c.N * self.sN + 64
        self.rsW = cols + c.res_pad
        self.rsH, self.rsD = self.OW * self.rsW, self.OH * self.OW * self.rsW
        self.rsN = self.OD * self.rsD
        self.res_len = c.res_off + c.N * self.rsN + 64
        self.kchunks = sum(s[5] for s in c.segs)
        self.w_pitch = 64 * self.kchunks
        self.w_K = self.w_pitch - c.w_trim if c.w_trim else 0
        self.w_rows = c.w_rows or c.cout
        self.w_gap = 3 if c.w_batched else 0          # NaN rows between weight batches
        self.nwb = c.N if c.w_batched else 1
        self.gn_slots, self.gn_slot0 = 4 * nsm + 2, 1
        self.n_tiles = cdiv(cols, 128)

    def footprint(self, c: Case):
        """Flat element indices [N, OD, OH, OW, cols] of the call's output."""
        n, d, h, w, k = np.ix_(np.arange(c.N), np.arange(self.OD), np.arange(self.OH), np.arange(self.OW),
                               np.arange(c.cols))
        return c.out_off + n * self.sN + d * self.sD + h * self.sH + w * self.sW + k


def make_operands(c: Case, g: Geom):
    """CPU tensors of every operand; the output, softmax-partial and GroupNorm buffers come prefilled."""
    gen = torch.Generator().manual_seed(zlib.crc32(c.name.encode()))
    rnd = lambda *s: torch.randn(*s, generator=gen)
    t = {}
    NA = 1 if c.a_broadcast else c.N
    for i, (ac, pitch) in enumerate(c.srcs):
        a = rnd(NA, *c.in_dhw, pitch)
        a[..., ac:] = float("nan")
        t[f"a{i}"] = a.to(ops.H16)
    K = sum(min(64, max(0, c.srcs[s[0]][0] - 64 * (s[4] + j))) for s in c.segs for j in range(s[5]))
    w = rnd(g.nwb, g.w_rows + g.w_gap, g.w_pitch) / K ** 0.5
    w[:, g.w_rows:] = float("nan")
    if g.w_K:
        w[..., g.w_K:] = float("nan")
    t["w"] = w.to(ops.H16)
    if c.bias:
        b = rnd(c.cout) * 0.5
        if c.huge:
            col = torch.arange(c.cout)
            b = torch.where(col % 3 == 0, b + 1e5, torch.where(col % 3 == 1, b - 1e5, b))
        t["bias"] = b
    if c.rowvec == "sample":
        t["rowvec"] = rnd(c.N, c.cout + 8) * 0.5
    elif c.rowvec == "bcast":
        t["rowvec"] = rnd(1, c.cout) * 0.5
    if c.row_bias:
        t["row_bias"] = rnd(g.OW) * 0.5
    if c.res:
        r = torch.full((g.res_len,), float("nan"))
        n, d, h, w_, k = np.ix_(np.arange(c.N), np.arange(g.OD), np.arange(g.OH), np.arange(g.OW), np.arange(c.cols))
        idx = torch.from_numpy((c.res_off + n * g.rsN + d * g.rsD + h * g.rsH + w_ * g.rsW + k).reshape(-1))
        r[idx] = rnd(idx.numel())
        t["res"] = r.to(ops.H16) if c.res == "h16" else r
    if c.out_f32:
        t["out"] = torch.full((g.out_len,), SENT32, dtype=torch.int32).view(torch.float32)
    else:
        t["out"] = torch.full((g.out_len,), SENT16, dtype=torch.int16).view(ops.H16)
    if c.stat:
        t["stat"] = torch.full((g.OW, g.n_tiles, 2), float("nan"))
    if c.gn:
        t["gn"] = torch.zeros(c.N, g.gn_slots, c.cout // c.gn, 2)
    return t


def fill(c: Case, g: Geom, ptr: dict) -> IgemmParams:
    """The parameter struct of case c over the buffers at `ptr` (name -> address, device or host alike)."""
    p = IgemmParams()
    for i, (ac, pitch) in enumerate(c.srcs):
        p.a_ptr[i], p.a_C[i], p.a_pitch[i] = ptr[f"a{i}"], ac, pitch
    p.in_N = c.N
    p.in_D, p.in_H, p.in_W = c.in_dhw
    p.stride_d, p.stride_h, p.stride_w = c.stride
    p.w_ptr, p.w_rows, p.w_pitch, p.w_K = ptr["w"], g.w_rows, g.w_pitch, g.w_K
    p.w_bstride = (g.w_rows + g.w_gap) * g.w_pitch if c.w_batched else 0
    p.w_batched, p.a_broadcast = int(c.w_batched), int(c.a_broadcast)
    p.n_seg = len(c.segs)
    for i, (src, dw, dh, dd, c0, nch) in enumerate(c.segs):
        s = p.seg[i]
        s.src, s.dw, s.dh, s.dd, s.c0, s.nchunks = src, dw, dh, dd, c0, nch
    esz = 4 if c.out_f32 else 2
    p.out_ptr = ptr["out"] + c.out_off * esz
    p.out_dtype = DT_F32 if c.out_f32 else DT_H16
    p.out_N, p.out_D, p.out_H, p.out_W = c.N, g.OD, g.OH, g.OW
    p.cout, p.out_cols = c.cout, c.cols
    p.out_sN, p.out_sD, p.out_sH, p.out_sW = g.sN, g.sD, g.sH, g.sW
    p.bias, p.row_bias = ptr.get("bias"), ptr.get("row_bias")
    if c.rowvec:
        p.rowvec = ptr["rowvec"]
        p.rowvec_bstride = c.cout + 8 if c.rowvec == "sample" else 0
    p.act1, p.scale, p.act2 = c.act1, c.scale, c.act2
    if c.res:
        p.res_dtype = DT_H16 if c.res == "h16" else DT_F32
        p.res_ptr = ptr["res"] + c.res_off * (2 if c.res == "h16" else 4)
        p.res_sN, p.res_sD, p.res_sH, p.res_sW = g.rsN, g.rsD, g.rsH, g.rsW
    p.stat_ptr = ptr.get("stat")
    if c.gn:
        p.gn_partial, p.gn_slots, p.gn_slot0, p.gn_group = ptr["gn"], g.gn_slots, g.gn_slot0, c.gn
    p.impl = c.impl
    return p


def host_ptrs(t):
    return {k: v.data_ptr() for k, v in t.items()}


def emulate(c: Case, g: Geom, t):
    """Run the emulator on copies of the CPU buffers; returns the buffers it wrote."""
    t = dict(t, out=t["out"].clone(), **{k: t[k].clone() for k in ("stat", "gn") if k in t})
    igemm_emulator.emulate(fill(c, g, host_ptrs(t)))
    return t


def bound(c: Case, g: Geom, t, got, want):
    """igemm_emulator.bound on the case's struct over the CPU operands."""
    return igemm_emulator.bound(fill(c, g, host_ptrs(t)), got, want, scale=c.scale)


# ------------------------------------------------------------------------------------------------------------------
# running a case
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    return _lib.require_device()


def launch(lib, c: Case, g: Geom, d, nsm):
    """One b200_igemm call on device buffers d; returns (rc, plan)."""
    p = fill(c, g, host_ptrs(d))
    ws = None
    if c.split:
        need = int(lib.b200_igemm_split_workspace_bytes(C.byref(p)))
        assert need > 0, "the planner does not split this call"
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        p.split_ws, p.split_ws_bytes = ws.data_ptr(), need
    plan = (C.c_int32 * 4)()
    assert lib.b200_igemm_plan(C.byref(p), nsm, int(c.split is not None), plan) == 0
    rc = lib.b200_igemm(C.byref(p), ops._stream())
    torch.cuda.synchronize()
    return rc, tuple(plan)[:2]


def to_device(t):
    return {k: v.cuda() for k, v in t.items()}


def run_case(lib, c: Case):
    nsm = int(lib.b200_sm_count())
    g = Geom(c, nsm)
    t = make_operands(c, g)
    ref = emulate(c, g, t)
    d = to_device(t)
    rc, plan = launch(lib, c, g, d, nsm)
    assert rc == 0, _lib.last_error()
    if c.expect is not None:
        assert plan == c.expect, f"{c.name} ran with (column tile, splits) = {plan}, not {c.expect}"
    got = {k: d[k].cpu() for k in ("out", "stat", "gn") if k in d}

    # footprint: nothing outside [N, OD, OH, OW] x [0, out_cols) at the call's strides was written
    bits = (lambda x: x.view(torch.int32).numpy()) if c.out_f32 else (lambda x: x.view(torch.int16).numpy())
    fp = g.footprint(c)
    outside = np.ones(g.out_len, dtype=bool)
    outside[fp.reshape(-1)] = False
    sent = SENT32 if c.out_f32 else SENT16
    assert (bits(got["out"])[outside] == sent).all(), f"{c.name}: stores outside the output footprint"

    # padding columns are +0
    ob = bits(got["out"])[fp]
    cv = c.cout // 2 if c.act1 == ACT_GEGLU else c.cout
    assert (ob[..., cv:] == 0).all(), f"{c.name}: padding columns are not +0"

    # values
    gv = got["out"].float().numpy()[fp].astype(np.float64)
    wv = ref["out"].float().numpy()[fp].astype(np.float64)
    assert np.isfinite(gv).all(), f"{c.name}: non-finite output"
    tol = bound(c, g, t, gv, wv)
    err = np.abs(gv - wv)
    if not (err <= tol).all():
        i = np.unravel_index(np.argmax(err - tol), err.shape)
        pytest.fail(f"{c.name}: got {gv[i]} want {wv[i]} at [n, d, h, w, col] = {i} (tol {tol[i]:.3g}); "
                    f"{int((err > tol).sum())} of {err.size} outside the bound")

    if c.gn:
        # relative to (sum |x|, sum x^2) + 1: fp32 partial sums of values that cancel (saturated +-65504) are only
        # accurate to that; a lost or misplaced tile is off by a few per cent of it
        gw = c.gn
        own = gv[..., :c.cout].reshape(c.N, -1, c.cout // gw, gw)
        want = np.stack([own.sum((1, 3)), (own * own).sum((1, 3))], -1)
        size = np.stack([np.abs(own).sum((1, 3)), (own * own).sum((1, 3))], -1) + 1
        gsum = got["gn"].double().numpy().sum(1)
        assert (np.abs(gsum - want) / size < 2e-4).all(), f"{c.name}: GroupNorm partials vs own output"
        emu = ref["gn"].double().numpy()[:, g.gn_slot0]
        assert (np.abs(gsum - emu) / size < 1e-3).all(), f"{c.name}: GroupNorm partials vs emulator"

    if c.stat:
        st = got["stat"].double().numpy()
        rows = gv.reshape(g.OW, c.cols)
        for ti in range(g.n_tiles):
            seg = rows[:, ti * 128:min((ti + 1) * 128, c.cout)]
            if seg.shape[1] == 0:
                assert (st[:, ti, 0] == -np.inf).all() and (st[:, ti, 1] == 0).all(), f"{c.name}: empty tile {ti}"
                continue
            mx = seg.max(1)
            assert (st[:, ti, 0] == mx).all(), f"{c.name}: softmax max of tile {ti}"
            s = np.exp(seg - mx[:, None]).sum(1)
            assert (np.abs(st[:, ti, 1] - s) <= 1e-5 * s).all(), f"{c.name}: softmax sum of tile {ti}"
        es = ref["stat"].double().numpy()
        fin = np.isfinite(es[..., 0])
        assert (fin == np.isfinite(st[..., 0])).all()
        assert np.allclose(st[fin], es[fin], rtol=1e-4, atol=1e-5), f"{c.name}: softmax partials vs emulator"

    # determinism: the same call again, on the same prefilled buffers
    d2 = to_device(t)
    rc2, _ = launch(lib, c, g, d2, nsm)
    assert rc2 == 0, _lib.last_error()
    assert (bits(d2["out"].cpu()) == bits(got["out"])).all(), f"{c.name}: a second call stores different bits"
    if c.stat:
        assert torch.equal(d2["stat"].cpu().view(torch.int32), got["stat"].view(torch.int32))
    if c.gn and c.impl != 1:            # the check kernel's partials are fp32 atomics
        assert torch.equal(d2["gn"].cpu().view(torch.int32), got["gn"].view(torch.int32))
    return gv, wv


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_igemm_matches_emulator(cuda_device, lib, case):
    run_case(lib, case)


@pytest.mark.parametrize("case", SATURATION, ids=[c.name for c in SATURATION])
def test_igemm_16bit_stores_saturate(cuda_device, lib, case):
    """fp16 stores clamp to +-65504 on every store path (and the GroupNorm partials describe the clamped values);
    bf16 stores round like the emulator.  run_case already compares against the emulator, which saturates exactly
    when the library's 16-bit type is fp16."""
    got, want = run_case(lib, case)
    big = np.abs(want) >= 65504 if FP16 else np.abs(want) > 65504
    assert big.sum() > 0, "the case does not leave the fp16 range"
    if FP16:
        assert (np.abs(got[big]) == 65504).all()


# ------------------------------------------------------------------------------------------------------------------
# argument checks: B200_EINVAL and nothing launched
# ------------------------------------------------------------------------------------------------------------------
_GN = conv("e_gn", "", (64, 1), 1, (1, 8, 8), [64], 64, gn=8)
_STAT = gemm("e_stat", "", (128, 1), 64, 64, 200, out_f32=True, stat=True)
_GEGLU = gemm("e_geglu", "", (128, 1), 64, 64, 128, act1=ACT_GEGLU)
_WIDE = conv("e_wide", "", (256, 1), 1, (1, 8, 8), [64], 256, impl=3)
REJECTED = [
    replace(_GN, name="gn_misaligned_out", out_off=1),
    replace(_GN, name="gn_f32_residual", res="f32"),
    replace(_STAT, name="stat_not_gemm_shaped_N2", N=2),
    conv("stat_not_gemm_shaped_conv", "", (128, 1), 1, (1, 4, 8), [64], 64, out_f32=True, stat=True),
    replace(_STAT, name="stat_check_kernel", impl=1),
    replace(_GEGLU, name="geglu_residual", res="h16"),
    replace(_GEGLU, name="geglu_scale", scale=2.0),
    replace(_GEGLU, name="geglu_padding_columns", out_cols=72),
    replace(_WIDE, name="wide_row_bias", row_bias=True),
    replace(_WIDE, name="wide_out_cols_past_cout", out_cols=264),
]


@pytest.mark.parametrize("case", REJECTED, ids=[c.name for c in REJECTED])
def test_igemm_rejects_outside_contract(cuda_device, lib, case):
    g = Geom(case, int(lib.b200_sm_count()))
    t = make_operands(case, g)
    d = to_device(t)
    p = fill(case, g, host_ptrs(d))
    assert lib.b200_igemm(C.byref(p), ops._stream()) == B200_EINVAL
    torch.cuda.synchronize()
    raw = torch.int32 if case.out_f32 else torch.int16
    assert torch.equal(d["out"].cpu().view(raw), t["out"].view(raw)), "a rejected call wrote its output"

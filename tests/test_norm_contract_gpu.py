"""The normalisation entry points on the GPU against tests/norm_emulator.py, the float64 reading of include/b200gen.h.
Every case builds its operands once as host tensors in the ABI layout, runs the emulator on them and the library on
device copies, and checks:

  values       every stored element (of the sampled rows, for the C3 level-0 tensor) and the affine table against the
               emulator's bound;
  footprint    outputs are prefilled with a NaN bit pattern and have trailing rows; only [N * spatial][C] changes and
               the pad channels [C, y_pitch) become +0;
  ignored      input pad channels (and the SPADE tensor past 2C) hold NaN; every output stays finite;
  determinism  a second identical call stores identical bits;
  arguments    calls outside the contract return B200_EINVAL and leave the output untouched.

Case names say which branch each case pins: the vector width (vec8 / vec4 / vec2 / vec1, chosen from channel counts,
pitches and base-pointer alignment), the fused kernel's register form (kreg2 / kreg4 / kreg8 / loop), channels per
group (cpg), two sources and straddling groups, the activation, and the offset regime kN: every value is drawn around
N standard deviations from zero, where statistics formed as E[x^2] - mean^2 from fp32 sums lose their digits.
"""
import ctypes as C
import math
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import B200_EINVAL, GnApplyParams, GnStatsParams
from tests import norm_emulator as E

pytestmark = pytest.mark.gpu

H16 = ops.H16
SENT16 = 0x7FFF                     # NaN in fp16 and bf16: "never written"
DT_F32 = 1                          # B200_DT_F32
NAN = float("nan")
ACTS = {"none": E.ACT_NONE, "silu": E.ACT_SILU, "leaky": E.ACT_LEAKYRELU, "leaky02": E.ACT_LEAKYRELU02}


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def bits(x):
    return x.view(torch.int16)


def sentinel(n):
    return torch.full((n,), SENT16, dtype=torch.int16).view(H16)


def ratio_report(entry, name, r):
    print(f"\nBOUND {entry} {name} max(err/tol) = {r:.3f}")


@pytest.fixture(scope="module")
def lib():
    return _lib.require_device()


def place(X, pitch, off=0, extra=2):
    """X [rows, c] -> flat NaN-filled h16 buffer of rows + extra rows of `pitch`, starting `off` elements in."""
    rows, c = X.shape
    buf = torch.full((off + (rows + extra) * pitch,), NAN, dtype=H16)
    buf[off:off + rows * pitch].view(rows, pitch)[:, :c] = X.to(H16)
    return buf


def check_values(name, want, got):
    ex = E.excess(want, got)
    if not (ex <= 1).all():
        i = tuple(int(j) for j in torch.nonzero(ex == ex.max())[0])
        pytest.fail(f"{name}: got {float(got[i])} want {float(want.out[i])} at {i} "
                    f"(tol {float(E.tolerance(want, got.double())[i]):.3g}); {int((ex > 1).sum())} of {ex.numel()} "
                    f"outside the bound")
    return float(ex.max())


def check_affine(name, want, got):
    ex = E.affine_excess(want, got.view(want.a.shape[0], -1, 2))
    if not (ex <= 1).all():
        i = tuple(int(j) for j in torch.nonzero(ex == ex.max())[0])
        pytest.fail(f"{name}: affine entry {i} is {got.view(want.a.shape[0], -1, 2)[i].tolist()}, want "
                    f"({float(want.a[i])}, {float(want.b[i])}) +- ({float(want.a_err[i]):.3g}, "
                    f"{float(want.b_err[i]):.3g})")
    return float(ex.max())


def check_output(name, out, off, n_rows, C, pitch, want):
    """Footprint, pads and values of an h16 output buffer written from element `off` on."""
    ob = bits(out[off:]).view(-1, pitch)
    assert (bits(out[:off]) == SENT16).all(), f"{name}: stores before the output pointer"
    assert (ob[n_rows:] == SENT16).all(), f"{name}: stores past the last row"
    assert (ob[:n_rows, C:] == 0).all(), f"{name}: pad channels are not +0"
    stored = out[off:].view(-1, pitch)[:n_rows].double()
    assert torch.isfinite(stored[:, :C]).all(), f"{name}: non-finite output (an ignored NaN input reached it?)"
    return check_values(name, want, stored)


# ------------------------------------------------------------------------------------------------------------------
# GroupNorm: b200_groupnorm_stats + _apply, b200_groupnorm_fused
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Gn:
    name: str
    N: int
    spatial: int
    C0: int
    groups: int
    C1: int = 0
    act: str = "silu"
    k: float = 0.0
    pad0: int = 8                 # x_pitch[i] = C_i + pad_i
    pad1: int = 8
    ypad: int = 8                 # y_pitch = C + ypad
    off: int = 0                  # element offset of every base pointer
    eps: float = 1e-5

    @property
    def C(self):
        return self.C0 + self.C1


STATS = [
    Gn("vec8_N1_C64_g32_silu", 1, 999, 64, 32),
    Gn("vec8_N3_two_sources_straddling_group_none", 3, 333, 24, 4, C1=40, act="none"),
    Gn("vec8_N2_instance_norm_leaky", 2, 517, 16, 16, act="leaky"),
    Gn("vec8_N2_y_pitch_own_pad_leaky02", 2, 700, 32, 8, C1=32, pad0=0, pad1=16, ypad=24, act="leaky02"),
    Gn("vec1_odd_channels_N3_cpg3", 3, 301, 12, 4, pad0=4, act="leaky"),
    Gn("vec1_misaligned_pointers_N2", 2, 250, 32, 8, off=1, act="none"),
    Gn("vec1_pitch_not_multiple_of_8_two_sources", 2, 400, 16, 4, C1=16, pad0=3, pad1=5, act="leaky02"),
    Gn("vec1_ypitch_not_multiple_of_8_apply", 1, 128, 32, 4, ypad=3),
    Gn("vec8_k0_N2_long_chains", 2, 40000, 64, 8),
    Gn("vec8_k10_N2_long_chains", 2, 40000, 64, 8, k=10),
    Gn("vec8_k100_N2_long_chains", 2, 40000, 64, 8, k=100),
    Gn("vec8_k256_N2_long_chains", 2, 40000, 64, 8, k=256),
    Gn("vec1_k256_odd_channels", 2, 5000, 24, 8, pad0=1, k=256, act="none"),
]

FUSED = [
    Gn("vec8_kreg2_cpg64", 2, 100, 128, 2),
    Gn("vec8_kreg4_cpg64_leaky", 2, 200, 128, 2, act="leaky"),
    Gn("vec8_kreg8_cpg64_none", 1, 500, 64, 1, act="none"),
    Gn("vec8_loop_cpg64_leaky02", 3, 3000, 128, 2, act="leaky02"),
    Gn("vec4_base_offset_8_bytes", 2, 300, 32, 4, pad0=4, ypad=4, off=4),
    Gn("vec2_base_offset_4_bytes", 2, 300, 32, 4, pad0=2, ypad=2, off=2, act="leaky"),
    Gn("vec1_base_offset_2_bytes", 2, 300, 32, 4, off=1, act="none"),
    Gn("vec8_cpg1_instance_norm", 2, 777, 16, 16),
    Gn("vec8_cpg24_idle_threads", 2, 600, 48, 2, act="leaky02"),
    Gn("vec8_cpg40_idle_threads", 1, 900, 80, 2),
    Gn("vec8_cpg96_idle_threads", 2, 300, 192, 2, act="none"),
    Gn("vec8_cpg4096", 1, 6, 4096, 1),
    Gn("vec8_two_sources_cpg16", 2, 400, 32, 4, C1=32, pad1=16, act="leaky"),
    Gn("vec8_spatial1_var0", 3, 1, 64, 4),
    Gn("vec1_cpg1_spatial_2pow20", 1, 1 << 20, 8, 8, pad0=1, act="none"),
    Gn("vec8_kreg2_k0", 2, 64, 64, 1, k=0),
    Gn("vec8_kreg2_k10", 2, 64, 64, 1, k=10),
    Gn("vec8_kreg2_k100", 2, 64, 64, 1, k=100),
    Gn("vec8_kreg2_k256", 2, 64, 64, 1, k=256),
    Gn("vec8_loop_k10", 1, 4096, 256, 8, k=10),
    Gn("vec8_loop_k100", 1, 4096, 256, 8, k=100),
    Gn("vec8_loop_k256", 1, 4096, 256, 8, k=256),
    Gn("vec1_loop_k256", 1, 4096, 32, 1, pad0=1, k=256, act="none"),
]


def gn_operands(c: Gn):
    g = gen(c.name)
    rows = c.N * c.spatial
    X = torch.randn(rows, c.C, generator=g) + c.k
    if c.spatial == 1:
        X[:] = 0.75                                         # every group constant: var = 0
    t = {"x0": place(X[:, :c.C0], c.C0 + c.pad0, c.off)}
    t["x1"] = place(X[:, c.C0:], c.C1 + c.pad1, c.off) if c.C1 else None
    t["gamma"] = 1 + 0.5 * torch.randn(c.C, generator=g)
    t["beta"] = 0.5 * torch.randn(c.C, generator=g)
    t["y"] = sentinel(c.off + (rows + 3) * (c.C + c.ypad))
    return t


def gn_emulate(c, t):
    x1 = t["x1"][c.off:] if c.C1 else None
    return E.groupnorm(t["x0"][c.off:], x1, c.C0, c.C1, c.C0 + c.pad0, c.C1 + c.pad1, c.N, c.spatial, c.groups,
                       c.eps, t["gamma"], t["beta"], ACTS[c.act], c.C + c.ypad)


def gn_params(c, d, act=None):
    sp, ap = GnStatsParams(), GnApplyParams()
    ptr = lambda k: d[k].data_ptr() + 2 * c.off if d.get(k) is not None else None
    for p in (sp, ap):
        p.x_ptr[0], p.x_ptr[1] = ptr("x0"), ptr("x1")
        p.x_C[0], p.x_C[1] = c.C0, c.C1
        p.x_pitch[0], p.x_pitch[1] = c.C0 + c.pad0, c.C1 + c.pad1
        p.N, p.spatial = c.N, c.spatial
    sp.groups, sp.eps = c.groups, c.eps
    sp.gamma, sp.beta = d["gamma"].data_ptr(), d["beta"].data_ptr()
    sp.partial = d["partial"].data_ptr() if "partial" in d else None
    sp.affine = d["affine"].data_ptr() if "affine" in d else None
    ap.affine = sp.affine
    ap.act = ACTS[c.act] if act is None else act
    ap.y_ptr, ap.y_pitch = ptr("y"), c.C + c.ypad
    return sp, ap


def to_dev(t):
    return {k: (v.cuda() if v is not None else None) for k, v in t.items()}


def stats_apply_call(lib, c, t):
    d = to_dev(t)
    ws = lib.b200_groupnorm_workspace_bytes(c.N, c.spatial, c.C)
    d["partial"] = torch.empty(ws // 4, dtype=torch.float32, device="cuda")
    d["affine"] = torch.full((c.N * c.C * 2 + 16,), NAN, dtype=torch.float32, device="cuda")
    sp, ap = gn_params(c, d)
    rc = lib.b200_groupnorm_stats(C.byref(sp), ops._stream())
    assert rc == 0, _lib.last_error()
    rc = lib.b200_groupnorm_apply(C.byref(ap), ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["affine"].cpu(), d["y"].cpu()


@pytest.mark.parametrize("case", STATS, ids=[c.name for c in STATS])
def test_groupnorm_stats_apply_match_emulator(cuda_device, lib, case):
    c = case
    t = gn_operands(c)
    want, aff = gn_emulate(c, t)
    affine, y = stats_apply_call(lib, c, t)
    assert torch.isnan(affine[c.N * c.C * 2:]).all(), f"{c.name}: stores past the affine table"
    ra = check_affine(c.name, aff, affine[:c.N * c.C * 2])
    ry = check_output(c.name, y, c.off, c.N * c.spatial, c.C, c.C + c.ypad, want)
    ratio_report("groupnorm_stats", c.name, ra)
    ratio_report("groupnorm_apply", c.name, ry)
    a2, y2 = stats_apply_call(lib, c, t)
    assert torch.equal(a2.view(torch.int32), affine.view(torch.int32)) and torch.equal(bits(y2), bits(y)), \
        f"{c.name}: a second call stores different bits"


def fused_call(lib, c, t):
    d = to_dev(t)
    sp, ap = gn_params(c, d)
    rc = lib.b200_groupnorm_fused(C.byref(sp), C.byref(ap), ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["y"].cpu()


@pytest.mark.parametrize("case", FUSED, ids=[c.name for c in FUSED])
def test_groupnorm_fused_matches_emulator(cuda_device, lib, case):
    c = case
    t = gn_operands(c)
    want, _ = gn_emulate(c, t)
    y = fused_call(lib, c, t)
    ratio_report("groupnorm_fused", c.name, check_output(c.name, y, c.off, c.N * c.spatial, c.C, c.C + c.ypad, want))
    assert torch.equal(bits(fused_call(lib, c, t)), bits(y)), f"{c.name}: a second call stores different bits"


def test_groupnorm_stats_c3_level0_sampled_rows(cuda_device, lib):
    """b200_groupnorm_stats + apply on the C3 level-0 tensor (1 x 160 x 224 x 160 x 256, 2.9 GB of fp16) at offset
    k = 100: 512 chunks of 11 200 voxels over 8 rows of threads, 1400 fp32 terms per thread.  The float64 moments are
    summed on the device; the values are checked on sampled rows."""
    N, S, Cc, G, k = 1, 160 * 224 * 160, 256, 32, 100.0
    gcuda = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn(S, Cc, generator=gcuda, device="cuda") + k).to(H16)
    s = torch.zeros(G, dtype=torch.float64, device="cuda")
    for r0 in range(0, S, 1 << 18):
        s += x[r0:r0 + (1 << 18)].double().view(-1, G, 8).sum((0, 2))
    mean = s / (S * 8)
    q = torch.zeros_like(s)
    for r0 in range(0, S, 1 << 18):
        q += ((x[r0:r0 + (1 << 18)].double().view(-1, G, 8) - mean[None, :, None]) ** 2).sum((0, 2))
    var = (q / (S * 8)).cpu()[None]
    mean = mean.cpu()[None]
    piv = x[0].view(G, 8)[:, 0].double().cpu()[None]
    g = gen("c3")
    gamma, beta = 1 + 0.5 * torch.randn(Cc, generator=g), 0.5 * torch.randn(Cc, generator=g)
    eps = 1e-6
    s2 = var + eps
    rstd = 1 / torch.sqrt(s2)
    off = (mean - piv).abs()
    aff = E.affine_table(mean, rstd, E.STAT_GN * (torch.sqrt(s2) + off), E.STAT_GN * rstd * (1 + off ** 2 / s2),
                         gamma, beta, G)
    y = torch.empty_like(x)
    ws = lib.b200_groupnorm_workspace_bytes(N, S, Cc)
    partial = torch.empty(ws // 4, dtype=torch.float32, device="cuda")
    affine = torch.empty(N * Cc * 2, dtype=torch.float32, device="cuda")
    gd, bd = gamma.cuda(), beta.cuda()
    sp, ap = GnStatsParams(), GnApplyParams()
    for p in (sp, ap):
        p.x_ptr[0], p.x_ptr[1] = x.data_ptr(), None
        p.x_C[0], p.x_C[1], p.x_pitch[0], p.x_pitch[1] = Cc, 0, Cc, 0
        p.N, p.spatial = N, S
    sp.groups, sp.eps, sp.gamma, sp.beta = G, eps, gd.data_ptr(), bd.data_ptr()
    sp.partial, sp.affine = partial.data_ptr(), affine.data_ptr()
    ap.affine, ap.act, ap.y_ptr, ap.y_pitch = affine.data_ptr(), E.ACT_SILU, y.data_ptr(), Cc
    assert lib.b200_groupnorm_stats(C.byref(sp), ops._stream()) == 0, _lib.last_error()
    assert lib.b200_groupnorm_apply(C.byref(ap), ops._stream()) == 0, _lib.last_error()
    torch.cuda.synchronize()
    ratio_report("groupnorm_stats", "c3_level0_k100", check_affine("c3_level0", aff, affine.cpu()))
    rows = torch.cat([torch.arange(64), torch.arange(S - 64, S), torch.arange(64, S - 64, 9973)]).cuda()
    X = x[rows].double().cpu()[None]
    want = E.gn_output(X, aff, E.ACT_SILU, Cc)
    got = y[rows].double().cpu()
    ratio_report("groupnorm_apply", "c3_level0_k100_sampled", check_values("c3_level0", want, got))
    del x, y, partial


# ------------------------------------------------------------------------------------------------------------------
# b200_groupnorm_from_partials_ex
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Part:
    name: str
    N: int
    spatial: int
    C0: int
    groups: int
    w0: int = 8
    slots0: int = 4
    C1: int = 0
    w1: int = 8
    slots1: int = 4
    k: float = 0.0


PARTIALS = [
    Part("w8_one_source_slots1", 2, 64, 64, 8, slots0=1),
    Part("w4_one_source_slots7", 3, 90, 128, 32, w0=4, slots0=7),
    Part("w8_w4_two_sources_slots5_3", 2, 120, 32, 6, C1=64, w1=4, slots0=5, slots1=3),
    Part("w4_w8_two_sources_cpg16_slots264", 1, 600, 32, 4, w0=4, C1=32, slots0=264, slots1=2),
    Part("w8_k10_slots132", 2, 2000, 64, 4, slots0=132, k=10),
]


def partial_operands(c: Part):
    g = gen(c.name)
    X = (torch.randn(c.N, c.spatial, c.C0 + c.C1, generator=g) + c.k).to(H16).double()
    parts = [E.partials_from(X[..., :c.C0], c.slots0, c.w0)]
    if c.C1:
        parts.append(E.partials_from(X[..., c.C0:], c.slots1, c.w1))
    gamma = 1 + 0.5 * torch.randn(c.C0 + c.C1, generator=g)
    beta = 0.5 * torch.randn(c.C0 + c.C1, generator=g)
    return X, parts, gamma, beta


def partials_call(lib, c, parts, gamma, beta, widths):
    d_parts = [p.reshape(-1).cuda() for p in parts]
    gd, bd = gamma.cuda(), beta.cuda()
    affine = torch.full((c.N * (c.C0 + c.C1) * 2 + 16,), NAN, dtype=torch.float32, device="cuda")
    sp = GnStatsParams()
    sp.x_ptr[0], sp.x_ptr[1] = None, None
    sp.x_C[0], sp.x_C[1] = c.C0, c.C1
    sp.N, sp.spatial, sp.groups, sp.eps = c.N, c.spatial, c.groups, 1e-5
    sp.gamma, sp.beta, sp.affine = gd.data_ptr(), bd.data_ptr(), affine.data_ptr()
    pp = (C.c_void_p * 2)(d_parts[0].data_ptr(), d_parts[1].data_ptr() if c.C1 else None)
    slots = (C.c_int32 * 2)(c.slots0, c.slots1 if c.C1 else 0)
    grp = (C.c_int32 * 2)(*widths)
    rc = lib.b200_groupnorm_from_partials_ex(C.byref(sp), pp, slots, grp, ops._stream())
    torch.cuda.synchronize()
    return rc, affine.cpu()


@pytest.mark.parametrize("case", PARTIALS, ids=[c.name for c in PARTIALS])
def test_groupnorm_from_partials_ex_matches_emulator(cuda_device, lib, case):
    c = case
    X, parts, gamma, beta = partial_operands(c)
    want = E.gn_from_partials([p.reshape(-1) for p in parts], [c.slots0, c.slots1], [c.w0, c.w1], c.C0, c.C1, c.N,
                              c.spatial, c.groups, 1e-5, gamma, beta)
    rc, affine = partials_call(lib, c, parts, gamma, beta, (c.w0, c.w1))
    assert rc == 0, _lib.last_error()
    assert torch.isnan(affine[c.N * (c.C0 + c.C1) * 2:]).all(), f"{c.name}: stores past the affine table"
    ratio_report("groupnorm_from_partials", c.name, check_affine(c.name, want, affine[:-16]))
    rc, again = partials_call(lib, c, parts, gamma, beta, (c.w0, c.w1))
    assert torch.equal(again.view(torch.int32), affine.view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# b200_spade_apply
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Spade:
    name: str
    N: int
    spatial: int
    C0: int
    C1: int = 0
    gb_extra: int = 8             # gb_pitch = 2C + gb_extra (NaN past 2C)
    pad: int = 8
    act: str = "leaky02"


SPADE = [
    Spade("vec8_N2_leaky02", 2, 500, 32),
    Spade("vec8_two_sources_gb_pitch_2C_plus_16_silu", 2, 300, 16, C1=24, gb_extra=16, act="silu"),
    Spade("vec8_gb_pitch_2C_none", 1, 64, 64, gb_extra=0, act="none"),
    Spade("scalar_odd_channels_leaky", 3, 101, 12, C1=4, pad=3, act="leaky"),
    Spade("scalar_gb_pitch_not_multiple_of_8", 2, 77, 16, gb_extra=3),
]


def spade_operands(c: Spade):
    g = gen(c.name)
    Cc, rows = c.C0 + c.C1, c.N * c.spatial
    gbp = 2 * Cc + c.gb_extra
    X = torch.randn(rows, Cc, generator=g)
    t = {"x0": place(X[:, :c.C0], c.C0 + c.pad), "x1": place(X[:, c.C0:], c.C1 + c.pad) if c.C1 else None,
         "gb": place(torch.randn(rows, 2 * Cc, generator=g), gbp),
         "ax": torch.randn(c.N, Cc, 2, generator=g), "gba": 0.5 * torch.randn(c.N, 2 * Cc, 2, generator=g),
         "y": sentinel((rows + 3) * (Cc + c.pad))}
    return t, gbp


def spade_call(lib, c, t, gbp, gb_pitch=None):
    d = to_dev(t)
    ap = GnApplyParams()
    ap.x_ptr[0], ap.x_ptr[1] = d["x0"].data_ptr(), d["x1"].data_ptr() if c.C1 else None
    ap.x_C[0], ap.x_C[1] = c.C0, c.C1
    ap.x_pitch[0], ap.x_pitch[1] = c.C0 + c.pad, c.C1 + c.pad
    ap.N, ap.spatial, ap.affine, ap.act = c.N, c.spatial, d["ax"].data_ptr(), ACTS[c.act]
    ap.y_ptr, ap.y_pitch = d["y"].data_ptr(), c.C0 + c.C1 + c.pad
    rc = lib.b200_spade_apply(C.byref(ap), d["gb"].data_ptr(), gbp if gb_pitch is None else gb_pitch,
                              d["gba"].data_ptr(), ops._stream())
    torch.cuda.synchronize()
    return rc, d["y"].cpu()


@pytest.mark.parametrize("case", SPADE, ids=[c.name for c in SPADE])
def test_spade_apply_matches_emulator(cuda_device, lib, case):
    c = case
    t, gbp = spade_operands(c)
    Cc = c.C0 + c.C1
    want = E.spade(t["x0"], t["x1"], c.C0, c.C1, c.C0 + c.pad, c.C1 + c.pad, c.N, c.spatial, t["ax"], t["gb"], gbp,
                   t["gba"], ACTS[c.act], Cc + c.pad)
    rc, y = spade_call(lib, c, t, gbp)
    assert rc == 0, _lib.last_error()
    ratio_report("spade_apply", c.name, check_output(c.name, y, 0, c.N * c.spatial, Cc, Cc + c.pad, want))
    assert torch.equal(bits(spade_call(lib, c, t, gbp)[1]), bits(y)), f"{c.name}: a second call stores different bits"


# ------------------------------------------------------------------------------------------------------------------
# b200_layernorm and the LayerNorm prologue of b200_rows_linear
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Ln:
    name: str
    M: int
    C: int
    xpad: int = 8
    ypad: int = 8
    k: float = 0.0
    g_off: int = 0                # element offset of gamma (4 bytes: not 16-byte aligned)


LAYERNORM = [
    Ln("vpl1_C8_M1", 1, 8),
    Ln("vpl1_C256_M9", 9, 256),
    Ln("vpl2_C264_M9", 9, 264),
    Ln("vpl2_C512", 33, 512),
    Ln("vpl4_C520", 17, 520),
    Ln("vpl4_C1024", 10, 1024),
    Ln("vpl8_C1032", 10, 1032),
    Ln("vpl8_C2048", 9, 2048),
    Ln("scalar_C2056_over_2048", 9, 2056),
    Ln("scalar_C100_not_multiple_of_8", 13, 100, xpad=4, ypad=5),
    Ln("scalar_misaligned_gamma", 11, 320, g_off=1),
    Ln("vpl1_C64_M100000", 100_000, 64),
    Ln("vpl2_C320_k10", 16, 320, k=10),
    Ln("vpl2_C320_k100", 16, 320, k=100),
    Ln("vpl2_C320_k256", 16, 320, k=256),
    Ln("scalar_C100_k256", 16, 100, xpad=1, k=256),
]


def ln_operands(c: Ln):
    g = gen(c.name)
    t = {"x": place(torch.randn(c.M, c.C, generator=g) + c.k, c.C + c.xpad),
         "gamma": torch.cat([torch.zeros(c.g_off), 1 + 0.5 * torch.randn(c.C, generator=g)]),
         "beta": 0.5 * torch.randn(c.C, generator=g),
         "y": sentinel((c.M + 3) * (c.C + c.ypad))}
    return t


def ln_call(lib, c, t):
    d = to_dev(t)
    rc = lib.b200_layernorm(d["x"].data_ptr(), c.M, c.C, c.C + c.xpad, d["gamma"].data_ptr() + 4 * c.g_off,
                            d["beta"].data_ptr(), 1e-5, d["y"].data_ptr(), c.C + c.ypad, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["y"].cpu()


@pytest.mark.parametrize("case", LAYERNORM, ids=[c.name for c in LAYERNORM])
def test_layernorm_matches_emulator(cuda_device, lib, case):
    c = case
    t = ln_operands(c)
    want = E.layernorm(t["x"], c.M, c.C, c.C + c.xpad, t["gamma"][c.g_off:], t["beta"], 1e-5, c.C + c.ypad)
    y = ln_call(lib, c, t)
    ratio_report("layernorm", c.name, check_output(c.name, y, 0, c.M, c.C, c.C + c.ypad, want))
    assert torch.equal(bits(ln_call(lib, c, t)), bits(y)), f"{c.name}: a second call stores different bits"


ROWS_LINEAR = [(8, 512, 0.0), (8, 512, 10.0), (8, 512, 100.0), (8, 512, 256.0), (1, 100, 0.0), (3, 1000, 100.0)]


@pytest.mark.parametrize("M,K,k", ROWS_LINEAR, ids=[f"M{m}_K{kk}_k{int(k)}" for m, kk, k in ROWS_LINEAR])
def test_rows_linear_layernorm_prologue_matches_emulator(cuda_device, lib, M, K, k):
    """An identity weight (O = K, fp32 out) returns the staged LayerNorm row exactly."""
    g = gen(f"rl{M}_{K}_{k}")
    xp, Kp = K + 8, (K + 7) // 8 * 8
    x = place(torch.randn(M, K, generator=g) + k, xp)
    gamma, beta = 1 + 0.5 * torch.randn(K, generator=g), 0.5 * torch.randn(K, generator=g)
    want = E.rows_linear_ln(x, M, K, xp, gamma, beta, 1e-5)
    W = torch.zeros(K, Kp, dtype=H16)
    W[:, :K] = torch.eye(K, dtype=H16)
    d = {"x": x.cuda(), "g": gamma.cuda(), "b": beta.cuda(), "w": W.cuda()}
    op = K + 4
    outs = []
    for _ in range(2):
        out = torch.full((M + 2, op), NAN, dtype=torch.float32, device="cuda")
        rc = lib.b200_rows_linear(d["x"].data_ptr(), xp, M, K, d["g"].data_ptr(), d["b"].data_ptr(), 1e-5,
                                  d["w"].data_ptr(), Kp, K, None, E.ACT_NONE, None, 0, out.data_ptr(), op,
                                  DT_F32, ops._stream())
        torch.cuda.synchronize()
        assert rc == 0, _lib.last_error()
        outs.append(out.cpu())
    o = outs[0]
    assert torch.isnan(o[M:]).all() and torch.isnan(o[:M, K:]).all(), "stores outside [M][O]"
    got = o[:M, :K].double()
    assert torch.equal(E.h16(got), got), "the staged row is not a 16-bit value"
    ratio_report("rows_linear_ln", f"M{M}_K{K}_k{int(k)}", check_values("rows_linear", want, got))
    assert torch.equal(outs[1].view(torch.int32), o.view(torch.int32))


# ------------------------------------------------------------------------------------------------------------------
# nearest resizing (b200_interpolate as ops.resize_nearest calls it)
# ------------------------------------------------------------------------------------------------------------------
RESIZE = [("2d_26x6_to_22x74", 2, 1, 26, 6, 1, 22, 74, 12), ("3d_14x6x26_to_46x74x22", 1, 14, 6, 26, 46, 74, 22, 8),
          ("3d_6x14x26_to_74x46x22_pitch3", 2, 6, 14, 26, 74, 46, 22, 3)]


@pytest.mark.parametrize("name,N,D,H,W,OD,OH,OW,pitch", RESIZE, ids=[r[0] for r in RESIZE])
def test_resize_nearest_through_interpolate_bit_exact(cuda_device, lib, name, N, D, H, W, OD, OH, OW, pitch):
    g = gen(name)
    x = torch.randn(N, D, H, W, pitch, generator=g).to(H16)
    x[..., pitch - 1] = 0.0 if pitch > 4 else x[..., pitch - 1]    # a pad channel: copied as it is
    ncd = x.float().permute(0, 4, 1, 2, 3)
    want = F.interpolate(ncd, size=(OD, OH, OW), mode="nearest").permute(0, 2, 3, 4, 1).to(H16)
    n = N * OD * OH * OW * pitch
    y = sentinel(n + 37).cuda()
    xd = ops.CL(x.cuda(), pitch, 3)
    ops._resample(xd, (OD, OH, OW), _lib.INTERPOLATE_NEAREST, y=y[:n].view(N, OD, OH, OW, pitch))
    torch.cuda.synchronize()
    y = y.cpu()
    assert (bits(y[n:]) == SENT16).all(), "stores past the output"
    assert torch.equal(bits(y[:n]), bits(want.reshape(-1))), f"{name}: differs from F.interpolate"
    got = ops.resize_nearest(xd, (OD, OH, OW)).t.cpu()
    assert torch.equal(bits(got.reshape(-1)), bits(y[:n])), f"{name}: ops.resize_nearest differs"


# ------------------------------------------------------------------------------------------------------------------
# argument checks: B200_EINVAL, output untouched
# ------------------------------------------------------------------------------------------------------------------
GN_REJECTED = [
    ("apply_relu", "apply", Gn("e_relu", 1, 16, 16, 4), E.ACT_RELU),
    ("apply_gelu", "apply", Gn("e_gelu", 1, 16, 16, 4), E.ACT_GELU),
    ("fused_relu", "fused", Gn("e_frelu", 1, 16, 16, 4), E.ACT_RELU),
    ("fused_gelu", "fused", Gn("e_fgelu", 1, 16, 16, 4), E.ACT_GELU),
    ("fused_straddling_group", "fused", Gn("e_strad", 1, 16, 12, 2, C1=4, pad0=4, pad1=4), None),
    ("fused_cpg_over_512_vectors", "fused", Gn("e_cpg", 1, 1, 4104, 1), None),
    ("fused_spatial_2pow24", "fused", Gn("e_sp", 1, 1 << 24, 8, 1, pad0=0, ypad=0), None),
    ("stats_C8192", "stats", Gn("e_c8192", 1, 2, 8192, 32, pad0=0, ypad=0), None),
]


@pytest.mark.parametrize("name,entry,case,act", GN_REJECTED, ids=[r[0] for r in GN_REJECTED])
def test_groupnorm_rejects_outside_contract(cuda_device, lib, name, entry, case, act):
    c = case
    t = gn_operands(c)
    d = to_dev(t)
    d["affine"] = torch.full((c.N * c.C * 2,), NAN, dtype=torch.float32, device="cuda")
    d["partial"] = torch.empty(lib.b200_groupnorm_workspace_bytes(c.N, c.spatial, c.C) // 4, device="cuda")
    sp, ap = gn_params(c, d, act=act)
    if entry == "apply":
        rc = lib.b200_groupnorm_apply(C.byref(ap), ops._stream())
    elif entry == "fused":
        rc = lib.b200_groupnorm_fused(C.byref(sp), C.byref(ap), ops._stream())
    else:
        rc = lib.b200_groupnorm_stats(C.byref(sp), ops._stream())
    torch.cuda.synchronize()
    assert rc == B200_EINVAL, (rc, _lib.last_error())
    assert torch.equal(bits(d["y"].cpu()), bits(t["y"])), "a rejected call wrote its output"
    assert torch.isnan(d["affine"].cpu()).all(), "a rejected call wrote the affine table"


def test_from_partials_rejects_two_channel_producer_groups(cuda_device, lib):
    c = Part("e_w2", 1, 16, 16, 4)
    X, parts, gamma, beta = partial_operands(c)
    rc, affine = partials_call(lib, c, parts, gamma, beta, (2, 0))
    assert rc == B200_EINVAL
    assert torch.isnan(affine).all(), "a rejected call wrote the affine table"


def test_spade_rejects_gb_pitch_below_2C(cuda_device, lib):
    c = Spade("e_gbp", 1, 8, 16)
    t, gbp = spade_operands(c)
    rc, y = spade_call(lib, c, t, gbp, gb_pitch=31)
    assert rc == B200_EINVAL
    assert torch.equal(bits(y), bits(t["y"])), "a rejected call wrote its output"

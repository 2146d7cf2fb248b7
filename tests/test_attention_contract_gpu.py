"""The attention entry points on the GPU against tests/attention_emulator.py, the float64 reading of include/b200gen.h.
Every case builds its operands once as host tensors in the ABI layout, runs the emulator on them and the library on
device copies, and checks:

  values       every stored element (of the sampled query rows, for the largest grids) against the emulator's bound;
  footprint    outputs are prefilled with a NaN bit pattern, have trailing rows and a pitch past heads * dh; only
               [B][T][heads * dh] (softmax: [M][p_pitch], pad columns +0) may change;
  ignored      q / k columns past heads * dh, key / value rows in [S, kv_rows) and after the last batch item, V^T
               columns [S, vt_pitch) and residual pad columns hold NaN; every output stays finite;
  determinism  a second identical call stores identical bits; the pos_dev forms store the bits of the host forms;
  arguments    calls outside the contract return B200_EINVAL and leave the output untouched.

Case names say which path they pin: head_dim (f64 / f128 / f256 / d512), T, S, batch B, heads h, "fused" (q and k
pitches of a fused projection, 3 * heads * dh), "res_own" (residual with its own pitch) or "res_packed" (the
output's), and the score regime: random at 1/sqrt(dh), scale 0 (keys past S would score exactly like valid ones),
negative scale, "peaked" (40/sqrt(dh): one key dominates, the rest underflow ex2's flush to zero) and "late" (a score
ramp along the keys, so the running maximum grows in every key block).  The d512 cases include a partner CTA without
rows (T < 64, odd tile counts), key blocks where consumer 1 has no valid key (S <= 64, S = 129) and a grid of 70
clusters (more than the 66 an H100 runs at once).
"""
import ctypes as C
import math
import zlib
from dataclasses import dataclass, replace

import pytest
import torch

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import B200_EINVAL, FlashParams
from tests import attention_emulator as E

pytestmark = pytest.mark.gpu

H16 = ops.H16
FP16 = H16 is torch.float16
SENT16 = 0x7FFF                     # NaN in fp16 and bf16: "never written"
NAN = float("nan")


def round8(n):
    return (n + 7) // 8 * 8


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def nan_rows(n, pitch, dtype=None):
    return torch.full((n * pitch,), NAN, dtype=dtype or H16)


def sentinel(n):
    return torch.full((n,), SENT16, dtype=torch.int16).view(H16)


def bits(x):
    return x.view(torch.int16)


def ratio_report(entry, name, r):
    print(f"\nBOUND {entry} {name} max(err/tol) = {r:.3f}")


@pytest.fixture(scope="module")
def lib():
    return _lib.require_device()


def check_values(name, want, got):
    ex = E.excess(want, got)
    if not (ex <= 1).all():
        i = tuple(int(j) for j in torch.nonzero(ex == ex.max())[0])
        pytest.fail(f"{name}: got {float(got[i])} want {float(want.out[i])} at {i} "
                    f"(tol {float(E.tolerance(want, got.double())[i]):.3g}); {int((ex > 1).sum())} of {ex.numel()} "
                    f"outside the bound")
    return float(ex.max())


# ------------------------------------------------------------------------------------------------------------------
# b200_attention_flash
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Flash:
    name: str
    dh: int
    T: int
    S: int
    B: int = 1
    heads: int = 1
    regime: str = "rand"          # rand / zero / neg / peaked / late / sat
    fused: bool = False           # q_pitch = k_pitch = 3 heads dh
    vt_pad: int = 8               # vt_pitch = round8(S) + vt_pad
    res: str | None = None        # "packed" (res_pitch = out_pitch) or "own" (a pitch of its own)

    @property
    def C(self):
        return self.heads * self.dh

    @property
    def scale(self):
        r = 1 / math.sqrt(self.dh)
        return {"zero": 0.0, "neg": -r, "peaked": 40 * r}.get(self.regime, r)

    def pitches(self):
        C = self.C
        qp = 3 * C if self.fused else C + 8
        kp = 3 * C if self.fused else C + 16
        op = C + 16
        rp = op if self.res == "packed" else C + 40
        return qp, kp, round8(self.S) + self.vt_pad, op, rp


FLASH = [
    Flash("f64_T1_S1", 64, 1, 1),
    Flash("f64_T63_S7_B2_h3_fused", 64, 63, 7, B=2, heads=3, fused=True),
    Flash("f64_T65_S65_B3_h2_res_own", 64, 65, 65, B=3, heads=2, res="own"),
    Flash("f64_T200_S1021_late_res_packed", 64, 200, 1021, regime="late", res="packed"),
    Flash("f64_T64_S129_h2_zero_scale", 64, 64, 129, heads=2, regime="zero"),
    Flash("f64_T128_S63_B2_neg_scale", 64, 128, 63, B=2, regime="neg", vt_pad=40),
    Flash("f64_T129_S127_h3_peaked", 64, 129, 127, heads=3, regime="peaked"),
    Flash("f128_T1_S64_h2", 128, 1, 64, heads=2),
    Flash("f128_T65_S129_B2_h3_fused_res_own", 128, 65, 129, B=2, heads=3, fused=True, res="own"),
    Flash("f128_T200_S1021_peaked", 128, 200, 1021, regime="peaked"),
    Flash("f128_T63_S65_zero_scale", 128, 63, 65, regime="zero"),
    Flash("f128_T257_S128_B3_late", 128, 257, 128, B=3, regime="late"),
    Flash("f256_T1_S7", 256, 1, 7),
    Flash("f256_T64_S65_B2_h2_res_own", 256, 64, 65, B=2, heads=2, res="own"),
    Flash("f256_T193_S1021_h3_fused_late", 256, 193, 1021, heads=3, fused=True, regime="late"),
    Flash("f256_T65_S64_zero_scale", 256, 65, 64, regime="zero"),
    Flash("f256_T129_S127_neg_res_packed", 256, 129, 127, regime="neg", res="packed"),
    Flash("f256_T70_S129_B3_peaked", 256, 70, 129, B=3, regime="peaked"),
    Flash("d512_T1_S1", 512, 1, 1),
    Flash("d512_T63_S64_h2_no_partner_rows", 512, 63, 64, heads=2),
    Flash("d512_T64_S7_B2", 512, 64, 7, B=2, res="own"),
    Flash("d512_T65_S129_B2_zero_scale", 512, 65, 129, B=2, regime="zero"),
    Flash("d512_T129_S65_zero_scale_odd_tiles", 512, 129, 65, regime="zero", res="own"),
    Flash("d512_T200_S1021_h2_fused_res_own", 512, 200, 1021, heads=2, fused=True, res="own"),
    Flash("d512_T4480_S127_h2_70_clusters", 512, 4480, 127, heads=2, res="packed"),
    Flash("d512_T130_S300_B3_late", 512, 130, 300, B=3, regime="late"),
    Flash("d512_T128_S128_peaked", 512, 128, 128, regime="peaked"),
    Flash("d512_T100_S200_neg_scale", 512, 100, 200, regime="neg", vt_pad=24),
]

# outputs past +-65504: fp16 stores clamp to +-65504 as the header states for h16 stores; bf16 rounds like the emulator
FLASH_SAT = [
    Flash("sat_f64_T65_S100", 64, 65, 100, heads=2, regime="sat", res="own"),
    Flash("sat_f128_T64_S64", 128, 64, 64, regime="sat", res="packed"),
    Flash("sat_f256_T1_S65", 256, 1, 65, regime="sat", res="own"),
    Flash("sat_d512_T65_S129", 512, 65, 129, regime="sat", res="own"),
]


def flash_operands(c: Flash):
    """Host buffers in the ABI layout: q [B][T][qp], k [B][S][kp], vt [B][C][vtp], res [B][T][rp], out [B][T][op],
    each with trailing rows; everything the call must not read is NaN, the output is the sentinel."""
    g = gen(c.name)
    rnd = lambda *s: torch.randn(*s, generator=g)
    B, T, S, Cc, dh = c.B, c.T, c.S, c.C, c.dh
    qp, kp, vtp, op, rp = c.pitches()
    Q, K, V = rnd(B, T, Cc), rnd(B, S, Cc), rnd(B, S, Cc)
    R = rnd(B, T, Cc)
    if c.regime == "late":              # channel 0 of every head: q = 2, k = 0.05 s -> the max grows along the keys
        for h in range(c.heads):
            Q[..., h * dh] = 2.0
            K[..., h * dh] = 0.05 * torch.arange(S, dtype=torch.float32)
    if c.regime == "sat":               # |o| ~ 100 on top of a residual of +-65504
        sign = 1.0 - 2.0 * (torch.arange(Cc) % 2)
        V = sign * (100 + rnd(B, S, Cc))
        R = sign * 65504.0 + 0 * R
    t = {}
    t["q"] = nan_rows(B * T + 2, qp)
    t["q"][:B * T * qp].view(B, T, qp)[..., :Cc] = Q.to(H16)
    t["k"] = nan_rows(B * S + 3, kp)
    t["k"][:B * S * kp].view(B, S, kp)[..., :Cc] = K.to(H16)
    t["vt"] = nan_rows(B * Cc + 2, vtp)
    t["vt"][:B * Cc * vtp].view(B, Cc, vtp)[..., :S] = V.transpose(1, 2).to(H16)
    if c.res:
        t["res"] = nan_rows(B * T + 2, rp)
        t["res"][:B * T * rp].view(B, T, rp)[..., :Cc] = R.to(H16)
    t["out"] = sentinel((B * T + 3) * op)
    return t


def flash_params(c: Flash, ptr, **over):
    qp, kp, vtp, op, rp = c.pitches()
    p = FlashParams()
    p.q, p.k, p.vt, p.out, p.res = ptr["q"], ptr["k"], ptr["vt"], ptr["out"], ptr.get("res")
    p.B, p.T, p.S, p.heads, p.dh = c.B, c.T, c.S, c.heads, c.dh
    p.q_pitch, p.k_pitch, p.vt_pitch, p.out_pitch = qp, kp, vtp, op
    p.res_pitch = rp if c.res else 0
    p.scale = c.scale
    for k, v in over.items():
        setattr(p, k, v)
    return p


def sample_rows(T):
    if T <= 512:
        return torch.arange(T)
    picked = set(range(64)) | set(range(T - 65, T)) | set(range(64, T, 37))
    return torch.tensor(sorted(picked))


def launch_flash(lib, c, t):
    d = {k: v.cuda() for k, v in t.items()}
    p = flash_params(c, {k: v.data_ptr() for k, v in d.items()})
    rc = lib.b200_attention_flash(C.byref(p), ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["out"].cpu()


def run_flash(lib, c: Flash):
    t = flash_operands(c)
    qp, kp, vtp, op, rp = c.pitches()
    rows = sample_rows(c.T)
    want = E.flash(t["q"], t["k"], t["vt"], t.get("res"), c.B, c.T, c.S, c.heads, c.dh, qp, kp, vtp, rp, c.scale,
                   rows=rows)
    out = launch_flash(lib, c, t)
    B, T, Cc = c.B, c.T, c.C
    ob = bits(out).view(-1, op)
    inside = torch.zeros_like(ob, dtype=torch.bool)
    inside[:B * T, :Cc] = True
    assert (ob[~inside] == SENT16).all(), f"{c.name}: stores outside [B][T][heads * dh]"
    stored = out.view(-1, op)[:B * T, :Cc]
    assert torch.isfinite(stored).all(), f"{c.name}: non-finite output (an ignored NaN input reached it?)"
    got = stored.view(B, T, Cc)[:, rows].double()
    r = check_values(c.name, want, got)
    assert torch.equal(bits(launch_flash(lib, c, t)), bits(out)), f"{c.name}: a second call stores different bits"
    return want, got, r


@pytest.mark.parametrize("case", FLASH, ids=[c.name for c in FLASH])
def test_flash_matches_emulator(cuda_device, lib, case):
    ratio_report("flash", case.name, run_flash(lib, case)[2])


@pytest.mark.parametrize("case", FLASH_SAT, ids=[c.name for c in FLASH_SAT])
def test_flash_16bit_stores_saturate(cuda_device, lib, case):
    want, got, r = run_flash(lib, case)
    ratio_report("flash", case.name, r)
    big = want.exact.abs() >= 65520
    assert big.sum() > 0, "the case does not leave the fp16 range"
    if FP16:
        assert (got[big].abs() == 65504).all()


# ------------------------------------------------------------------------------------------------------------------
# ops.attention's unfused path: score GEMM + softmax_rows_partials + PV GEMM
# ------------------------------------------------------------------------------------------------------------------
UNFUSED = [
    Flash("unfused_d192_B2_h2_T150_S100_res", 192, 150, 100, B=2, heads=2, res="own"),
    Flash("unfused_d768_B2_T70_S201_res", 768, 70, 201, B=2, res="packed"),
    Flash("unfused_forced_d128_B2_h2_T90_S77_res", 128, 90, 77, B=2, heads=2, res="own"),
]


@pytest.mark.parametrize("case", UNFUSED, ids=[c.name for c in UNFUSED])
def test_unfused_attention_matches_emulator(cuda_device, lib, case, monkeypatch):
    monkeypatch.setattr(ops, "_FORCE_UNFUSED_ATTENTION", True)
    c = case
    t = flash_operands(c)
    qp, kp, vtp, op, rp = c.pitches()
    B, T, S, Cc = c.B, c.T, c.S, c.C
    want = E.unfused(t["q"], t["k"], t["vt"], t["res"], B, T, S, c.heads, c.dh, qp, kp, vtp, rp, c.scale)
    q = t["q"].cuda()[:B * T * qp].view(B, T, qp)[..., :Cc]
    k = t["k"].cuda()[:B * S * kp].view(B, S, kp)[..., :Cc]
    vt = t["vt"].cuda()[:B * Cc * vtp].view(B, Cc, vtp)
    res = t["res"].cuda()[:B * T * rp].view(B, T, rp)
    out = ops.attention(q, k, None, c.heads, c.dh, c.scale, vt=vt, residual=res)
    out2 = ops.attention(q, k, None, c.heads, c.dh, c.scale, vt=vt, residual=res)
    torch.cuda.synchronize()
    got = out.cpu()[..., :Cc].double()
    assert torch.isfinite(got).all()
    assert (bits(out.cpu())[..., Cc:] == 0).all(), "pad columns are not +0"
    ratio_report("unfused", c.name, check_values(c.name, want, got))
    assert torch.equal(bits(out2.cpu()), bits(out.cpu())), f"{c.name}: a second call stores different bits"


# ------------------------------------------------------------------------------------------------------------------
# b200_attention_small(_ex) and b200_attention_decode
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Small:
    name: str
    dh: int
    T: int
    S: int
    B: int = 1
    heads: int = 1
    kv_rows: int = 0              # 0: S
    causal: int = 0
    q_pos0: int = 0
    pos: bool = False             # also run the pos_dev form (q_pos0 = *pos, S = *pos + T)

    @property
    def C(self):
        return self.heads * self.dh

    @property
    def kv(self):
        return self.kv_rows or self.S

    def pitches(self):           # odd pitches: the CUDA-core kernels read scalars
        C = self.C
        return C + 3, C + 5, C + 7, C + 9


SMALL = [
    Small("small_d1_B2_h3", 1, 5, 9, B=2, heads=3),
    Small("small_d3_h2_S1", 3, 4, 1, heads=2),
    Small("small_d32_B2_h2_causal_kv_rows", 32, 6, 10, B=2, heads=2, kv_rows=16, causal=1, q_pos0=4),
    Small("small_d33_B3_h2_kv_rows", 33, 3, 20, B=3, heads=2, kv_rows=29),
    Small("small_d64_B2_h2_S1000", 64, 3, 1000, B=2, heads=2),
    Small("small_d100_B2_causal_pos_dev", 100, 2, 9, B=2, kv_rows=12, causal=1, q_pos0=7, pos=True),
    Small("small_d256_B2_S64", 256, 5, 64, B=2),
    Small("small_d300_h2_causal_q_pos0", 300, 4, 33, heads=2, causal=1, q_pos0=29),
    Small("small_d1000_B2_S17", 1000, 3, 17, B=2),
    Small("small_d64_T1_S1_pos_dev", 64, 1, 1, B=2, heads=2, kv_rows=4, causal=1, pos=True),
]

DECODE = [
    Small("decode_d1_S1_B2_h3", 1, 1, 1, B=2, heads=3, kv_rows=4),
    Small("decode_d33_S3_h2", 33, 1, 3, heads=2, kv_rows=16),
    Small("decode_d64_S8_B3", 64, 1, 8, B=3, kv_rows=10),
    Small("decode_d200_S9_h2", 200, 1, 9, heads=2, kv_rows=9),
    Small("decode_d256_S1000_B2", 256, 1, 1000, B=2, kv_rows=1003),
    Small("decode_d64_S13_B2_h2_pos_dev", 64, 1, 13, B=2, heads=2, kv_rows=20, pos=True),
]


def small_operands(c: Small, q_rows):
    g = gen(c.name)
    rnd = lambda *s: torch.randn(*s, generator=g)
    qp, kp, vp, op = c.pitches()
    B, S, kv, Cc = c.B, c.S, c.kv, c.C
    t = {"q": nan_rows(q_rows + 2, qp), "k": nan_rows(B * kv + 2, kp), "v": nan_rows(B * kv + 2, vp)}
    t["q"][:q_rows * qp].view(q_rows, qp)[:, :Cc] = rnd(q_rows, Cc).to(H16)
    for name, pitch in (("k", kp), ("v", vp)):
        t[name][:B * kv * pitch].view(B, kv, pitch)[:, :S, :Cc] = rnd(B, S, Cc).to(H16)
    t["out"] = sentinel((q_rows + 3) * op)
    return t


def check_rows_footprint(name, out, n_rows, pitch, C):
    ob = bits(out).view(-1, pitch)
    inside = torch.zeros_like(ob, dtype=torch.bool)
    inside[:n_rows, :C] = True
    assert (ob[~inside] == SENT16).all(), f"{name}: stores outside the call's rows / columns"
    stored = out.view(-1, pitch)[:n_rows, :C]
    assert torch.isfinite(stored).all(), f"{name}: non-finite output"
    return stored


def small_call(lib, c, d, pos_dev=None):
    qp, kp, vp, op = c.pitches()
    S = 1 if pos_dev is not None else c.S
    rc = lib.b200_attention_small_ex(d["q"].data_ptr(), d["k"].data_ptr(), d["v"].data_ptr(), d["out"].data_ptr(), c.B,
                                     c.T, S, c.heads, c.dh, qp, kp, vp, op, 1 / math.sqrt(c.dh), c.kv, c.causal,
                                     c.q_pos0, pos_dev, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["out"].cpu()


@pytest.mark.parametrize("case", SMALL, ids=[c.name for c in SMALL])
def test_attention_small_matches_emulator(cuda_device, lib, case):
    c = case
    if c.pos:
        assert c.S == c.q_pos0 + c.T
    t = small_operands(c, c.B * c.T)
    qp, kp, vp, op = c.pitches()
    want = E.small(t["q"], t["k"], t["v"], c.B, c.T, c.S, c.heads, c.dh, qp, kp, vp, 1 / math.sqrt(c.dh), c.kv,
                   c.causal, c.q_pos0)
    out = small_call(lib, c, {k: v.cuda() for k, v in t.items()})
    got = check_rows_footprint(c.name, out, c.B * c.T, op, c.C).view(c.B, c.T, c.C).double()
    ratio_report("attention_small", c.name, check_values(c.name, want, got))
    assert torch.equal(bits(small_call(lib, c, {k: v.cuda() for k, v in t.items()})), bits(out))
    if c.dh <= 256 and not c.causal and c.kv == c.S:       # the plain entry point is the _ex form with these defaults
        d = {k: v.cuda() for k, v in t.items()}
        rc = lib.b200_attention_small(d["q"].data_ptr(), d["k"].data_ptr(), d["v"].data_ptr(), d["out"].data_ptr(),
                                      c.B, c.T, c.S, c.heads, c.dh, qp, kp, vp, op, 1 / math.sqrt(c.dh), ops._stream())
        torch.cuda.synchronize()
        assert rc == 0 and torch.equal(bits(d["out"].cpu()), bits(out))
    if c.pos:
        pos = torch.tensor([c.q_pos0], dtype=torch.int32, device="cuda")
        outp = small_call(lib, c, {k: v.cuda() for k, v in t.items()}, pos_dev=pos.data_ptr())
        assert torch.equal(bits(outp), bits(out)), f"{c.name}: the pos_dev form stores different bits"


def decode_call(lib, c, d, pos_dev=None):
    qp, kp, vp, op = c.pitches()
    rc = lib.b200_attention_decode(d["q"].data_ptr(), d["k"].data_ptr(), d["v"].data_ptr(), d["out"].data_ptr(), c.B,
                                   1 if pos_dev is not None else c.S, c.heads, c.dh, qp, kp, vp, op,
                                   1 / math.sqrt(c.dh), c.kv, pos_dev, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["out"].cpu()


@pytest.mark.parametrize("case", DECODE, ids=[c.name for c in DECODE])
def test_attention_decode_matches_emulator(cuda_device, lib, case):
    c = case
    t = small_operands(c, c.B)
    qp, kp, vp, op = c.pitches()
    want = E.decode(t["q"], t["k"], t["v"], c.B, c.S, c.heads, c.dh, qp, kp, vp, 1 / math.sqrt(c.dh), c.kv)
    out = decode_call(lib, c, {k: v.cuda() for k, v in t.items()})
    got = check_rows_footprint(c.name, out, c.B, op, c.C).double()
    ratio_report("attention_decode", c.name, check_values(c.name, want, got))
    assert torch.equal(bits(decode_call(lib, c, {k: v.cuda() for k, v in t.items()})), bits(out))
    if c.pos:
        pos = torch.tensor([c.S - 1], dtype=torch.int32, device="cuda")
        outp = decode_call(lib, c, {k: v.cuda() for k, v in t.items()}, pos_dev=pos.data_ptr())
        assert torch.equal(bits(outp), bits(out)), f"{c.name}: the pos_dev form stores different bits"


# ------------------------------------------------------------------------------------------------------------------
# b200_softmax_rows_partials
# ------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Softmax:
    name: str
    M: int
    S: int
    s_pitch: int
    p_pitch: int
    s_off: int = 0                # element offset of the score pointer (misaligned: the scalar path)


SOFTMAX = [
    Softmax("partials_float4_S1001_tail", 9, 1001, 1004, 1008),
    Softmax("partials_float4_S7_M300", 300, 7, 8, 8),
    Softmax("partials_scalar_odd_s_pitch", 10, 130, 131, 136),
    Softmax("partials_scalar_p_pitch_not_4", 4, 257, 260, 258),
    Softmax("partials_scalar_misaligned_scores", 6, 203, 204, 208, s_off=1),
]


def softmax_operands(c: Softmax):
    g = gen(c.name)
    x = torch.randn(c.M, c.S, generator=g) * 3
    x[0] = 1.5                                      # a constant row
    if c.M > 1:
        x[1] = torch.where(torch.arange(c.S) % 3 == 0, 1e4, -1e4)
    s = torch.full((c.s_off + (c.M + 1) * c.s_pitch,), NAN)
    s[c.s_off:c.s_off + c.M * c.s_pitch].view(c.M, c.s_pitch)[:, :c.S] = x
    # the igemm stat_ptr contract: (max, sum exp(v - max)) per 128-column tile of the fp32 row, plus a trailing tile
    # without columns, (-inf, 0)
    nt = (c.S + 127) // 128 + 1
    part = torch.zeros(c.M, nt, 2)
    xd = x.double()
    for i in range(nt):
        seg = xd[:, i * 128:min((i + 1) * 128, c.S)]
        if seg.shape[1] == 0:
            part[:, i, 0], part[:, i, 1] = -math.inf, 0.0
            continue
        mx = seg.amax(1)
        part[:, i, 0], part[:, i, 1] = mx.float(), torch.exp(seg - mx[:, None]).sum(1).float()
    return {"s": s, "out": sentinel((c.M + 2) * c.p_pitch), "part": part.reshape(-1)}


def softmax_call(lib, c, t):
    d = {k: v.cuda() for k, v in t.items()}
    sp = d["s"].data_ptr() + 4 * c.s_off
    rc = lib.b200_softmax_rows_partials(sp, c.M, c.S, c.s_pitch, d["part"].data_ptr(), d["part"].numel() // (2 * c.M),
                                        d["out"].data_ptr(), c.p_pitch, ops._stream())
    torch.cuda.synchronize()
    assert rc == 0, _lib.last_error()
    return d["out"].cpu()


@pytest.mark.parametrize("case", SOFTMAX, ids=[c.name for c in SOFTMAX])
def test_softmax_rows_match_emulator(cuda_device, lib, case):
    c = case
    t = softmax_operands(c)
    nt = t["part"].numel() // (2 * c.M)
    want = E.softmax_rows_partials(t["s"][c.s_off:], c.M, c.S, c.s_pitch, t["part"], nt, c.p_pitch)
    out = softmax_call(lib, c, t)
    ob = bits(out).view(-1, c.p_pitch)
    assert (ob[c.M:] == SENT16).all(), f"{c.name}: stores past row M"
    assert (ob[:c.M, c.S:] == 0).all(), f"{c.name}: pad columns are not +0"
    got = out.view(-1, c.p_pitch)[:c.M].double()
    ratio_report("partials", c.name, check_values(c.name, want, got))
    assert torch.equal(bits(softmax_call(lib, c, t)), bits(out)), f"{c.name}: a second call stores different bits"


# ------------------------------------------------------------------------------------------------------------------
# argument checks: B200_EINVAL, output untouched
# ------------------------------------------------------------------------------------------------------------------
_F = Flash("e_flash", 64, 64, 64, res="own")
FLASH_REJECTED = [
    ("dh_96", replace(_F, dh=96), {}),
    ("q_pitch_not_multiple_of_8", _F, {"q_pitch": 68}),
    ("vt_pitch_not_multiple_of_8", _F, {"vt_pitch": 76}),
    ("misaligned_k", _F, {"k": 2}),
    ("T_0", _F, {"T": 0}),
    ("heads_0", _F, {"heads": 0}),
    ("res_pitch_not_multiple_of_8", _F, {"res_pitch": 100}),
]


@pytest.mark.parametrize("name,case,over", FLASH_REJECTED, ids=[r[0] for r in FLASH_REJECTED])
def test_flash_rejects_outside_contract(cuda_device, lib, name, case, over):
    t = flash_operands(case)
    d = {k: v.cuda() for k, v in t.items()}
    ptr = {k: v.data_ptr() for k, v in d.items()}
    if "k" in over:
        ptr["k"] += over.pop("k")
    p = flash_params(case, ptr, **over)
    assert lib.b200_attention_flash(C.byref(p), ops._stream()) == B200_EINVAL
    torch.cuda.synchronize()
    assert torch.equal(bits(d["out"].cpu()), bits(t["out"])), "a rejected call wrote its output"


def test_attention_small_ex_rejects_kv_rows_below_S(cuda_device, lib):
    c = Small("e_small", 32, 2, 9, kv_rows=9)
    t = small_operands(c, 2)
    d = {k: v.cuda() for k, v in t.items()}
    qp, kp, vp, op = c.pitches()
    rc = lib.b200_attention_small_ex(d["q"].data_ptr(), d["k"].data_ptr(), d["v"].data_ptr(), d["out"].data_ptr(), 1, 2,
                                     9, 1, 32, qp, kp, vp, op, 0.2, 8, 0, 0, None, ops._stream())
    torch.cuda.synchronize()
    assert rc == B200_EINVAL
    assert torch.equal(bits(d["out"].cpu()), bits(t["out"])), "a rejected call wrote its output"


def test_attention_decode_rejects_head_dim_over_256(cuda_device, lib):
    c = Small("e_decode", 300, 1, 5, kv_rows=5)
    t = small_operands(c, 1)
    d = {k: v.cuda() for k, v in t.items()}
    qp, kp, vp, op = c.pitches()
    rc = lib.b200_attention_decode(d["q"].data_ptr(), d["k"].data_ptr(), d["v"].data_ptr(), d["out"].data_ptr(), 1, 5,
                                   1, 300, qp, kp, vp, op, 0.05, 5, None, ops._stream())
    torch.cuda.synchronize()
    assert rc == B200_EINVAL
    assert torch.equal(bits(d["out"].cpu()), bits(t["out"])), "a rejected call wrote its output"

"""The elementwise, scheduler and vector-quantiser entry points on the GPU against tests/elementwise_emulator.py, the
float64 reading of include/b200gen.h.  Every case builds its operands as host tensors in the ABI layout, runs the
emulator on them and the library on device copies, and checks:

  values       every stored element against the emulator's bound (copies and exact fp32 sequences bit for bit);
  footprint    outputs are prefilled with a NaN bit pattern, start after a leading offset and have trailing rows; only
               the written region changes and pad columns become +0 where the header says so;
  ignored      input columns the entry point must not read hold NaN; the outputs stay finite;
  determinism  a second identical call stores identical bits (not ddpm_kl's sample_sum or VQ's sqerr_sum: fp64 atomics
               in an unspecified order).

Argument checks run without a GPU in tests/test_elementwise_args_cpu.py.  Case names say which branch each case
pins: vector or scalar paths (picked by counts, pitches and pointer alignment), grid-stride passes over the capped grid
and scalar tails, prediction types and variance modes, the two VQ kernels and their tails.
"""
import ctypes as C
import math
import zlib
from types import SimpleNamespace as NS

import pytest
import torch
import torch.nn.functional as F  # noqa: F401

from generativemodels_b200 import _lib, ops
from generativemodels_b200._lib import DdimCoef, DdpmCoef, KlCoef, PndmCoef
from tests import elementwise_emulator as E

pytestmark = pytest.mark.gpu

H16 = ops.H16
SENT16 = 0x7FFF                     # NaN in fp16 and bf16: "never written"
NAN = float("nan")
F64 = torch.float64
DT_H16, DT_F32 = 0, 1


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def bits(x):
    return x.view(torch.int16) if x.element_size() == 2 else x.view(torch.int32) if x.element_size() == 4 else \
        x.view(torch.int64)


def sentinel16(n):
    return torch.full((n,), SENT16, dtype=torch.int16).view(H16)


def sentinel32(n):
    return torch.full((n,), NAN, dtype=torch.float32)


def ratio_report(entry, name, r):
    print(f"\nBOUND {entry} {name} max(err/tol) = {r:.3f}")


@pytest.fixture(scope="module")
def lib():
    return _lib.require_device()


def stream():
    return ops._stream()


def sync_ok(rc):
    torch.cuda.synchronize()
    assert rc == 0, (rc, _lib.last_error())


def check_values(name, want, got):
    ex = E.excess(want, got)
    if not (ex <= 1).all():
        i = tuple(int(j) for j in torch.nonzero(ex == ex.max())[0])
        pytest.fail(f"{name}: got {float(got[i])} want {float(want.out[i])} at {i} "
                    f"(tol {float(E.tolerance(want, got.double())[i]):.3g}); {int((ex > 1).sum())} of {ex.numel()} "
                    f"outside the bound")
    return float(ex.max())


def check_region(name, buf, off, n, want, pitch=None):
    """buf (host copy of an output prefilled with NaN) written from element `off` on: [off, off + n) holds the result,
    everything else still NaN.  Returns max err/tol."""
    assert torch.isnan(buf[:off].float()).all(), f"{name}: stores before the output pointer"
    assert torch.isnan(buf[off + n:].float()).all(), f"{name}: stores past the output"
    got = buf[off:off + n].double()
    return check_values(name, want, got.view(want.out.shape))


def h16_of(x):
    x = x.float()
    return (x.clamp(-65504, 65504) if H16 is torch.float16 else x).to(H16)


def nan_rows(X, pitch, extra=0, dtype=None):
    """X [rows, c] -> flat NaN-filled buffer of rows + extra rows of `pitch` (dtype: X's)."""
    rows, c = X.shape
    buf = torch.full(((rows + extra) * pitch,), NAN, dtype=dtype or X.dtype)
    buf[:rows * pitch].view(rows, pitch)[:, :c] = X
    return buf


# ------------------------------------------------------------------------------------------------------------------
# layout conversion
# ------------------------------------------------------------------------------------------------------------------
LAYOUT = [  # name, N, C, spatial, pitch, scale
    ("N1_C3_S999_pitch8", 1, 3, 999, 8, 1.0),
    ("N3_C5_S1000_pitch64_pitch_much_larger_than_C", 3, 5, 1000, 64, 1.0),
    ("N2_C40_S77_two_channel_tiles", 2, 40, 77, 48, 1.0),
    ("N1_C256_S1024", 1, 256, 1024, 256, 1.0),
    ("N2_C7_S33_saturating", 2, 7, 33, 8, 1e5),
]


@pytest.mark.parametrize("name,n,Cc,S,pitch,scale", LAYOUT, ids=[c[0] for c in LAYOUT])
def test_layout_conversion_bit_exact(cuda_device, lib, name, n, Cc, S, pitch, scale):
    g = gen(name)
    x = (scale * torch.randn(n * Cc * S, generator=g)).float()
    want = E.nchw_to_nhwc(x, n, Cc, S, pitch)
    xd = x.cuda()                                            # held: a freed temporary's memory can be reused
    outs = []
    for _ in range(2):
        y = sentinel16(8 + n * S * pitch + 3 * pitch).cuda()
        rc = lib.b200_nchw_to_nhwc(xd.data_ptr(), n, Cc, S, y[8:].data_ptr(), pitch, stream())
        sync_ok(rc)
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y)), f"{name}: a second call stores different bits"
    assert (bits(y[:8]) == SENT16).all() and (bits(y[8 + n * S * pitch:]) == SENT16).all(), f"{name}: footprint"
    got = y[8:8 + n * S * pitch].view(n * S, pitch)
    assert torch.equal(bits(got), bits(want.out.to(H16))), f"{name}: nchw_to_nhwc differs"
    if scale > 1 and H16 is torch.float16:
        assert got.float().abs().max() == 65504 and torch.isfinite(got.float()).all(), "fp16 stores must saturate"
    # back, from the 16-bit rows with NaN pads, and from fp32 rows with NaN pads
    rows = got.clone()
    rows[:, Cc:] = NAN
    for dt, src in ((DT_H16, rows), (DT_F32, (torch.randn(n * S, pitch, generator=g)).float())):
        src = src.clone()
        src[:, Cc:] = NAN
        back = E.nhwc_to_nchw(src.reshape(-1), n, Cc, S, pitch)
        y, sd = sentinel32(n * Cc * S + 40).cuda(), src.cuda()
        rc = lib.b200_nhwc_to_nchw(sd.data_ptr(), dt, n, Cc, S, pitch, y.data_ptr(), stream())
        sync_ok(rc)
        y = y.cpu()
        assert torch.isnan(y[n * Cc * S:]).all(), f"{name}: nhwc_to_nchw stores past the output"
        assert torch.equal(y[:n * Cc * S].double(), back.out), f"{name}: nhwc_to_nchw (dtype {dt}) differs"


# ------------------------------------------------------------------------------------------------------------------
# nearest x2 and the 2x average pool (b200_interpolate as ops calls it), axpy_h16
# ------------------------------------------------------------------------------------------------------------------
RESAMPLE = [  # name, N, D, H, W, C, pitch, dims, scale
    ("dims2_N2_C16_5x6", 2, 1, 5, 6, 16, 16, 2, 1.0),
    ("dims2_three_slices_odd_7x9_pitch24", 1, 3, 7, 9, 20, 24, 2, 1.0),
    ("dims3_N1_C24_3x4x5", 1, 3, 4, 5, 24, 24, 3, 1.0),
    ("dims3_odd_5x7x9_N3_pitch16", 3, 5, 7, 9, 9, 16, 3, 1.0),
    ("dims3_large_values", 1, 4, 6, 8, 8, 8, 3, 3e4),
]


@pytest.mark.parametrize("name,n,D,H,W,Cc,pitch,dims,scale", RESAMPLE, ids=[c[0] for c in RESAMPLE])
def test_nearest2x_avgpool2_through_interpolate_bit_exact(cuda_device, lib, name, n, D, H, W, Cc, pitch, dims, scale):
    g = gen(name)
    X = torch.zeros(n * D * H * W, pitch)
    X[:, :Cc] = scale * torch.randn(n * D * H * W, Cc, generator=g)
    x = h16_of(X).view(n, D, H, W, pitch)                    # pad channels 0: every channel is processed
    xd = ops.CL(x.cuda(), Cc, dims)
    ncd = x.double().permute(0, 4, 1, 2, 3)
    if dims == 2:                                            # D slices, each resampled in 2-D
        ncd = ncd.transpose(1, 2).reshape(n * D, pitch, H, W)
    up = F.interpolate(ncd, scale_factor=2.0, mode="nearest")
    pool = (F.avg_pool3d if dims == 3 else F.avg_pool2d)(ncd, 2, 2)
    even = [D if dims == 2 else D // 2 * 2, H // 2 * 2, W // 2 * 2]           # AvgPool's floor windows
    for entry, fn, want, mode, src in (("upsample_nearest2x", ops.upsample_nearest2x, up, _lib.INTERPOLATE_NEAREST, None),
                                       ("avgpool2", ops.avgpool2, pool, _lib.INTERPOLATE_AREA, even)):
        if dims == 2:
            want = want.reshape(n, D, pitch, *want.shape[2:]).transpose(1, 2)
        want = E.h16(want.permute(0, 2, 3, 4, 1))
        outs = []
        for _ in range(2):
            y = sentinel16(want.numel() + 5 * pitch).cuda()
            ops._resample(xd, want.shape[1:4], mode, src, y[:want.numel()].view(want.shape))
            torch.cuda.synchronize()
            outs.append(y.cpu())
        y = outs[0]
        assert torch.equal(bits(outs[1]), bits(y)), f"{name}: {entry} repeats differ"
        assert (bits(y[want.numel():]) == SENT16).all(), f"{name}: {entry} stores past the output"
        assert torch.equal(bits(y[:want.numel()]), bits(want.reshape(-1).to(H16))), f"{name}: {entry} differs"
        assert torch.equal(bits(fn(xd).t.cpu().reshape(-1)), bits(y[:want.numel()])), f"{name}: ops.{entry} differs"
        ratio_report(entry, name, 0.0)


AXPY = [("n8", 8, 0.75, 1.0), ("n4096_alpha_neg", 4096, -1.5, 1.0), ("n1000008", 1_000_008, 0.3, 1.0),
        ("saturating", 64, 1.0, 4e4)]


@pytest.mark.parametrize("name,n,alpha,scale", AXPY, ids=[c[0] for c in AXPY])
def test_axpy_h16_matches_emulator(cuda_device, lib, name, n, alpha, scale):
    g = gen(name)
    a, b = h16_of(scale * torch.randn(n, generator=g)), h16_of(scale * torch.randn(n, generator=g))
    if scale > 1:
        a[:8], b[:8] = h16_of(torch.full((8,), 6e4)), h16_of(torch.full((8,), 6e4))
    want = E.axpy_h16(a, b, alpha, n)
    ad, bd = a.cuda(), b.cuda()
    outs = []
    for _ in range(2):
        y = sentinel16(n + 64).cuda()
        sync_ok(lib.b200_axpy_h16(ad.data_ptr(), bd.data_ptr(), alpha, y.data_ptr(), n, stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    assert (bits(y[n:]) == SENT16).all(), "stores past n"
    if scale > 1 and H16 is torch.float16:
        assert (y[:8].float() == 65504).all(), "fp16 stores must saturate"
    ratio_report("axpy_h16", name, check_values(name, want, y[:n].double()))


# ------------------------------------------------------------------------------------------------------------------
# copy_channels, geglu
# ------------------------------------------------------------------------------------------------------------------
COPY = [  # name, C, src_pitch, dst_pitch, dst_off, rows, base offset (elements) of src / dst
    ("vec8_C16_off8", 16, 24, 40, 8, 1000, 0),
    ("vec8_C64_off0", 64, 64, 128, 0, 333, 0),
    ("scalar_C5_off3", 5, 8, 16, 3, 777, 0),
    ("scalar_C16_misaligned_base", 16, 24, 40, 8, 100, 1),
    ("scalar_pitch_not_multiple_of_8", 8, 12, 20, 8, 50, 0),
]


@pytest.mark.parametrize("name,Cc,sp,dp,off,rows,base", COPY, ids=[c[0] for c in COPY])
def test_copy_channels_bit_exact(cuda_device, lib, name, Cc, sp, dp, off, rows, base):
    g = gen(name)
    src = torch.cat([torch.zeros(base, dtype=H16), nan_rows(h16_of(torch.randn(rows, Cc, generator=g)), sp)])
    want = E.copy_channels(src[base:], Cc, sp, rows).out
    dst0 = sentinel16(base + (rows + 2) * dp)
    sd = src.cuda()
    outs = []
    for _ in range(2):
        d = dst0.cuda()
        sync_ok(lib.b200_copy_channels(sd.data_ptr() + 2 * base, Cc, sp, d.data_ptr() + 2 * base, dp, off, rows,
                                       stream()))
        outs.append(d.cpu())
    d = outs[0]
    assert torch.equal(bits(outs[1]), bits(d))
    body = d[base:].view(-1, dp)
    assert (bits(d[:base]) == SENT16).all() and (bits(body[rows:]) == SENT16).all(), f"{name}: footprint"
    rest = torch.cat([body[:rows, :off], body[:rows, off + Cc:]], 1)
    assert (bits(rest) == SENT16).all(), f"{name}: the rest of the destination row was touched"
    assert torch.equal(bits(body[:rows, off:off + Cc]), bits(want.to(H16))), f"{name}: copy differs"


GEGLU = [("M1_H8", 1, 8, 16, 8), ("M77_H40_x_pitch_96_y_pitch_48", 77, 40, 96, 48), ("M4096_H1280", 4096, 1280, 2560, 1280),
         ("M5_H16_large", 5, 16, 40, 24)]


@pytest.mark.parametrize("name,M,H,xp,yp", GEGLU, ids=[c[0] for c in GEGLU])
def test_geglu_matches_emulator(cuda_device, lib, name, M, H, xp, yp):
    g = gen(name)
    scale = 300.0 if name.endswith("large") else 2.0
    x = nan_rows(h16_of(scale * torch.randn(M, 2 * H, generator=g)), xp)
    want = E.geglu(x, M, H, xp)
    xd = x.cuda()
    outs = []
    for _ in range(2):
        y = sentinel16((M + 2) * yp).cuda()
        sync_ok(lib.b200_geglu(xd.data_ptr(), M, H, xp, y.data_ptr(), yp, stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    body = y.view(-1, yp)
    assert (bits(body[M:]) == SENT16).all() and (bits(body[:M, H:]) == SENT16).all(), f"{name}: footprint"
    assert torch.isfinite(body[:M, :H].float()).all() or scale > 2
    ratio_report("geglu", name, check_values(name, want, body[:M, :H].double()))


# ------------------------------------------------------------------------------------------------------------------
# tap_gather, tap_sum
# ------------------------------------------------------------------------------------------------------------------
TAPS = [  # name, N, D, H, W, kd, kh, kw, pd, ph, pw, stride, C (gather) / cout (sum)
    ("conv_in_3d_C1_40x36x44", 1, 40, 36, 44, 3, 3, 3, 1, 1, 1, 1, 1),
    ("conv_in_2d_C3_200x190", 2, 1, 200, 190, 1, 3, 3, 0, 1, 1, 1, 3),
    ("conv_in_3d_C2_stride2_65x60x81", 2, 65, 60, 81, 3, 3, 3, 1, 1, 1, 2, 2),
    ("aniso_3x1x2_pad101_C3", 2, 9, 10, 11, 3, 1, 2, 1, 0, 1, 1, 3),
    ("aniso_2x3x1_pad020_C4_stride2", 1, 8, 9, 7, 2, 3, 1, 0, 2, 0, 2, 4),
]
SUMS = [
    ("out_3d_cout1_40x36x44", 1, 40, 36, 44, 3, 3, 3, 1, 1, 1, 1, 1),
    ("out_2d_cout3_200x190", 2, 1, 200, 190, 1, 3, 3, 0, 1, 1, 1, 3),
    ("out_3d_cout4_20x30x61", 1, 20, 30, 61, 3, 3, 3, 1, 1, 1, 1, 4),
    ("aniso_3x1x2_pad101_cout2", 2, 9, 10, 11, 3, 1, 2, 1, 0, 1, 1, 2),
    ("aniso_1x3x2_pad012_cout3_no_bias", 1, 6, 9, 8, 1, 3, 2, 0, 1, 2, 1, 3),
]


def tap_geom(n, D, H, W, kd, kh, kw, pd, ph, pw, s):
    OD, OH, OW = ((e + 2 * p - k) // s + 1 for e, p, k in ((D, pd, kd), (H, ph, kh), (W, pw, kw)))
    return [n, D, H, W, OD, OH, OW, kd, kh, kw, s, s, s, pd, ph, pw]


@pytest.mark.parametrize("case", TAPS, ids=[c[0] for c in TAPS])
def test_tap_gather_bit_exact(cuda_device, lib, case):
    name, *gm, Cc = case
    geom = tap_geom(*gm)
    g = gen(name)
    rows_in = geom[0] * geom[1] * geom[2] * geom[3]
    xp = Cc + 3
    x = nan_rows(h16_of(torch.randn(rows_in, Cc, generator=g)), xp)
    taps = geom[7] * geom[8] * geom[9]
    op = (taps * Cc + 7) // 8 * 8 + 8
    want = E.tap_gather(x, Cc, xp, geom, op).out
    V = want.shape[0]
    xd, gd = x.cuda(), (C.c_int32 * 16)(*geom)
    outs = []
    for _ in range(2):
        y = sentinel16((V + 3) * op).cuda()
        sync_ok(lib.b200_tap_gather(xd.data_ptr(), Cc, xp, gd, y.data_ptr(), op, stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    assert (bits(y[V * op:]) == SENT16).all(), f"{name}: stores past the last row"
    assert torch.equal(bits(y[:V * op].view(V, op)), bits(want.to(H16))), f"{name}: tap_gather differs"


@pytest.mark.parametrize("out_h16", [True, False], ids=["h16_out", "f32_out"])
@pytest.mark.parametrize("case", SUMS, ids=[c[0] for c in SUMS])
def test_tap_sum_matches_emulator(cuda_device, lib, case, out_h16):
    name, *gm, cout = case
    geom = tap_geom(*gm)
    g = gen(name)
    taps = geom[7] * geom[8] * geom[9]
    rows_in = geom[0] * geom[1] * geom[2] * geom[3]
    yp = taps * cout + 4
    y = nan_rows(torch.randn(rows_in, taps * cout, generator=g).float(), yp)
    bias = None if name.endswith("no_bias") else torch.randn(cout, generator=g).float()
    op = 8
    want = E.tap_sum(y, yp, geom, cout, bias, op, out_h16)
    V = want.out.shape[0]
    yd, gd = y.cuda(), (C.c_int32 * 16)(*geom)
    bd = bias.cuda() if bias is not None else None
    outs = []
    for _ in range(2):
        o = (sentinel16 if out_h16 else sentinel32)((V + 2) * op).cuda()
        sync_ok(lib.b200_tap_sum(yd.data_ptr(), yp, gd, cout, bd.data_ptr() if bd is not None else None, o.data_ptr(),
                                 op, DT_H16 if out_h16 else DT_F32, stream()))
        outs.append(o.cpu())
    o = outs[0]
    assert torch.equal(bits(outs[1]), bits(o))
    assert torch.isnan(o[V * op:].float()).all(), f"{name}: stores past the last row"
    body = o[:V * op].view(V, op)
    assert (bits(body[:, cout:]) == 0).all(), f"{name}: pad columns are not +0"
    ratio_report("tap_sum", f"{name}_{'h16' if out_h16 else 'f32'}", check_values(name, want, body.double()))


# ------------------------------------------------------------------------------------------------------------------
# embed_tokens, cache_append, advance_i32, vq_gather
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_pos_dev", [False, True], ids=["host_pos0", "pos_dev"])
def test_embed_tokens_bit_exact(cuda_device, lib, use_pos_dev):
    g = gen(f"emb{use_pos_dev}")
    V, L, Cc, pitch, seq, M, pos0 = 50, 40, 24, 32, 7, 21, 5
    tok = torch.randint(0, V, (M,), generator=g)
    te, pe = torch.randn(V * Cc, generator=g).float(), torch.randn(L * Cc, generator=g).float()
    want = E.embed_tokens(tok, M, seq, pos0, te, pe, Cc, pitch).out
    d = [t.cuda() for t in (tok, te, pe)]
    pos = torch.tensor([pos0], dtype=torch.int32).cuda()
    outs = []
    for _ in range(2):
        y = sentinel16((M + 2) * pitch).cuda()
        sync_ok(lib.b200_embed_tokens(d[0].data_ptr(), M, seq, 0 if use_pos_dev else pos0, d[1].data_ptr(),
                                      d[2].data_ptr(), Cc, y.data_ptr(), pitch,
                                      pos.data_ptr() if use_pos_dev else None, stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    assert (bits(y[M * pitch:]) == SENT16).all()
    assert torch.equal(bits(y[:M * pitch].view(M, pitch)), bits(want.to(H16)))


CACHE = [("pos0", 0), ("pos_middle", 9), ("rows_past_L_dropped", 14), ("all_past_L", 16), ("negative_pos", -2),
         ("all_negative", -5)]


@pytest.mark.parametrize("name,pos", CACHE, ids=[c[0] for c in CACHE])
def test_cache_append_drops_rows_outside_the_cache(cuda_device, lib, name, pos):
    """The cache sits inside a larger NaN buffer: a store at a row before 0 or at / past L lands in the same allocation
    and shows in the footprint."""
    g = gen(name)
    B, T, L, pitch, guard = 3, 4, 16, 24, 4 * 16 * 24
    src = h16_of(torch.randn(B * T * pitch, generator=g))
    cache = h16_of(torch.randn(B * L * pitch, generator=g))
    want = E.cache_append(src, cache, B, T, L, pitch, pos).out
    buf = torch.cat([sentinel16(guard), cache, sentinel16(guard)]).cuda()
    p = torch.tensor([pos], dtype=torch.int32).cuda()
    sd = src.cuda()
    sync_ok(lib.b200_cache_append(sd.data_ptr(), buf[guard:].data_ptr(), B, T, L, pitch, p.data_ptr(),
                                  stream()))
    buf = buf.cpu()
    assert (bits(buf[:guard]) == SENT16).all() and (bits(buf[-guard:]) == SENT16).all(), f"{name}: stored outside"
    assert torch.equal(bits(buf[guard:-guard]), bits(want.to(H16))), f"{name}: cache differs"
    sync_ok(lib.b200_advance_i32(p.data_ptr(), T, stream()))
    sync_ok(lib.b200_advance_i32(p.data_ptr(), -1, stream()))
    assert int(p.item()) == pos + T - 1


def test_vq_gather_bit_exact_and_clamps(cuda_device, lib):
    g = gen("vqg")
    M, K, D, qp = 1000, 37, 13, 24
    idx = torch.randint(0, K, (M,), generator=g)
    idx[:4] = torch.tensor([-5, -1, K, K + 100])
    cb = torch.randn(K * D, generator=g).float()
    want = E.vq_gather(idx, M, cb, K, D, qp).out
    y = sentinel16((M + 2) * qp).cuda()
    idd, cd = idx.cuda(), cb.cuda()
    sync_ok(lib.b200_vq_gather(idd.data_ptr(), M, cd.data_ptr(), K, D, y.data_ptr(), qp, stream()))
    y = y.cpu()
    assert (bits(y[M * qp:]) == SENT16).all()
    assert torch.equal(bits(y[:M * qp].view(M, qp)), bits(want.to(H16)))


# ------------------------------------------------------------------------------------------------------------------
# timestep_embedding, small_linear
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 2, 32, 33, 256, 320, 1281])
def test_timestep_embedding_matches_emulator(cuda_device, lib, dim):
    t = torch.tensor([0.0, 1.0, 7.5, 250.0, 999.0, 1000.0], dtype=torch.float32)
    n = t.numel()
    want = E.timestep_embedding(t, n, dim, 10000.0)
    td = t.cuda()
    outs = []
    for _ in range(2):
        y = sentinel32(n * dim + 33).cuda()
        sync_ok(lib.b200_timestep_embedding(td.data_ptr(), n, dim, 10000.0, y.data_ptr(), stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    ratio_report("timestep_embedding", f"dim{dim}", check_region(f"dim{dim}", y, 0, n * dim, want))
    if dim % 2:
        assert (bits(y[:n * dim].view(n, dim)[:, -1]) == 0).all(), "odd dim: the last column is not +0"


LINEAR = [  # name, M, K, O, act_in, act_out, bias, base offset (floats) of x
    ("vec_K384_M2_silu_none", 2, 384, 300, E.ACT_SILU, E.ACT_NONE, True, 0),
    ("vec_K1024_M1_silu_silu", 1, 1024, 1280, E.ACT_SILU, E.ACT_SILU, True, 0),
    ("vec_K2176_M3_none_gelu", 3, 2176, 77, E.ACT_NONE, E.ACT_GELU, True, 0),
    ("vec_K1024_M64_relu_tanh_no_bias", 64, 1024, 40, E.ACT_RELU, E.ACT_TANH, False, 0),
    ("scalar_K100_M3_silu_silu", 3, 100, 70, E.ACT_SILU, E.ACT_SILU, True, 0),
    ("scalar_K100_M1_leaky_sigmoid", 1, 100, 9, E.ACT_LEAKYRELU, E.ACT_SIGMOID, True, 0),
    ("scalar_K100_M64_gelu_leaky02_no_bias", 64, 100, 33, E.ACT_GELU, E.ACT_LEAKYRELU02, False, 0),
    ("scalar_K384_misaligned_x_tanh_relu", 2, 384, 50, E.ACT_TANH, E.ACT_RELU, True, 1),
    ("scalar_K128_sigmoid_none", 5, 128, 16, E.ACT_SIGMOID, E.ACT_NONE, True, 2),
    ("vec_K128_M4096_none_silu", 4096, 128, 8, E.ACT_NONE, E.ACT_SILU, True, 0),
]


@pytest.mark.parametrize("name,M,K,O,ai,ao,has_b,base", LINEAR, ids=[c[0] for c in LINEAR])
def test_small_linear_matches_emulator(cuda_device, lib, name, M, K, O, ai, ao, has_b, base):
    g = gen(name)
    x = torch.cat([torch.zeros(base), 2 * torch.randn(M * K, generator=g)]).float()
    W = (torch.randn(O * K, generator=g) / math.sqrt(K)).float()
    b = torch.randn(O, generator=g).float() if has_b else None
    want = E.small_linear(x[base:], M, K, W, b, O, ai, ao)
    xd, wd = x.cuda(), W.cuda()
    bd = b.cuda() if has_b else None
    outs = []
    for _ in range(2):
        y = sentinel32(M * O + 17).cuda()
        sync_ok(lib.b200_small_linear(xd.data_ptr() + 4 * base, M, K, wd.data_ptr(), bd.data_ptr() if has_b else None,
                                      O, ai, ao, y.data_ptr(), stream()))
        outs.append(y.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y))
    ratio_report("small_linear", name, check_region(name, y, 0, M * O, E.Result(
        want.exact.reshape(-1), want.out.reshape(-1), want.err.reshape(-1), "f32")))


# ------------------------------------------------------------------------------------------------------------------
# scheduler steps
# ------------------------------------------------------------------------------------------------------------------
def f32v(v):
    return float(torch.tensor(v, dtype=torch.float32))


def ddim_struct(pred, clip, sigma):
    c = DdimCoef()
    c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t = math.sqrt(0.3), math.sqrt(0.7)
    c.sqrt_alpha_prod_prev, c.sigma = math.sqrt(0.55), sigma
    c.dir_coef = math.sqrt(1 - 0.55 - sigma ** 2)
    c.clip_min, c.clip_max, c.prediction_type, c.clip = -1.0, 1.0, pred, clip
    return c


def threads_cap(lib):
    return 16 * lib.b200_sm_count() * 256


DDIM = [  # name, n or callable(lib), pred, clip, noise, x0, misaligned (elements) of one pointer
    ("vec_n2pow24_plus3_capped_grid_passes_tail", lambda lib: (1 << 24) + 3, E.PRED_EPSILON, 0, True, True, 0),
    ("vec_n_8x256x1000_two_vectors_per_thread", lambda lib: 8 * 256 * 1000, E.PRED_V, 1, False, True, 0),
    ("vec_n_minus_4_last_thread_single", lambda lib: 8 * 256 * 1000 - 4, E.PRED_SAMPLE, 1, True, False, 0),
    ("vec_n_plus_4_one_vector_threads", lambda lib: 8 * 256 * 1000 + 4, E.PRED_EPSILON, 1, True, True, 0),
    ("vec_n_capped_4x_threads_plus_4", lambda lib: 4 * threads_cap(lib) + 4, E.PRED_V, 0, True, True, 0),
    ("vec_n_capped_4x_threads_minus_4", lambda lib: 4 * threads_cap(lib) - 4, E.PRED_SAMPLE, 0, False, False, 0),
    ("scalar_model_out_4_bytes_off", lambda lib: 100_003, E.PRED_EPSILON, 0, True, True, 1),
    ("scalar_noise_4_bytes_off_v_clip", lambda lib: 4099, E.PRED_V, 1, True, True, 2),
    ("vec_n1", lambda lib: 1, E.PRED_V, 0, True, True, 0),
    ("vec_n7_tail_only", lambda lib: 7, E.PRED_SAMPLE, 1, True, True, 0),
]


@pytest.mark.parametrize("name,nf,pred,clip,noise,want_x0,mis", DDIM, ids=[c[0] for c in DDIM])
def test_ddim_step_matches_emulator(cuda_device, lib, name, nf, pred, clip, noise, want_x0, mis):
    n = nf(lib)
    g = gen(name)
    m, s, z = (torch.randn(n, generator=g) for _ in range(3))
    c = ddim_struct(pred, clip, 0.2 if noise else 0.0)
    rp, rx = E.ddim_step(m, s, z if noise else None, c, n)
    dev = []
    for i, t in enumerate((m, s, z)):
        off = 1 if (mis == 1 and i == 0) or (mis == 2 and i == 2) else 0
        buf = torch.cat([torch.zeros(off), t]).cuda()
        dev.append((buf, 4 * off))
    ptr = lambda i: dev[i][0].data_ptr() + dev[i][1]
    outs = []
    for _ in range(2):
        prev, x0 = sentinel32(n + 37).cuda(), sentinel32(n + 37).cuda()
        sync_ok(lib.b200_ddim_step(ptr(0), ptr(1), ptr(2) if noise else None, C.byref(c), prev.data_ptr(),
                                   x0.data_ptr() if want_x0 else None, n, stream()))
        outs.append((prev.cpu(), x0.cpu()))
    (prev, x0), (p2, x2) = outs
    assert torch.equal(bits(p2), bits(prev)) and torch.equal(bits(x2), bits(x0))
    ratio_report("ddim_step", name, check_region(name, prev, 0, n, rp))
    if want_x0:
        ratio_report("ddim_step_x0", name, check_region(name, x0, 0, n, rx))
    else:
        assert torch.isnan(x0).all(), "pred_x0 == NULL but something was stored"


def ddpm_struct(pred, var_mode, clip):
    c = DdpmCoef()
    a_t, a_prev, beta = 0.4, 0.45, 0.02
    var = (1 - a_prev) / (1 - a_t) * beta
    c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t = math.sqrt(a_t), math.sqrt(1 - a_t)
    c.coef_x0, c.coef_xt = math.sqrt(a_prev) * beta / (1 - a_t), math.sqrt(1 - beta) * (1 - a_prev) / (1 - a_t)
    c.sigma, c.clip_min, c.clip_max, c.min_log, c.max_log = math.sqrt(var), -1.0, 1.0, var, beta
    c.var_mode, c.prediction_type, c.clip = var_mode, pred, clip
    return c


DDPM = [  # name, pred, var_mode, clip, noise
    ("fixed_eps_noise", E.PRED_EPSILON, 0, 1, True),
    ("fixed_eps_t0_noise_null", E.PRED_EPSILON, 0, 1, False),
    ("learned_sample", E.PRED_SAMPLE, 1, 0, True),
    ("learned_range_v_clip", E.PRED_V, 2, 1, True),
    ("learned_range_eps_t0_noise_null", E.PRED_EPSILON, 2, 0, False),
]


@pytest.mark.parametrize("name,pred,vm,clip,noise", DDPM, ids=[c[0] for c in DDPM])
def test_ddpm_step_matches_emulator(cuda_device, lib, name, pred, vm, clip, noise):
    n = 200_003
    g = gen(name)
    m, s, z, pv = (torch.randn(n, generator=g) for _ in range(4))
    pv = (0.01 * pv.abs()) if vm == 1 else pv.tanh()
    c = ddpm_struct(pred, vm, clip)
    rp, rx = E.ddpm_step(m, s, z if noise else None, pv, c, n)
    d = [t.cuda() for t in (m, s, z, pv)]
    outs = []
    for _ in range(2):
        prev, x0 = sentinel32(n + 9).cuda(), sentinel32(n + 9).cuda()
        sync_ok(lib.b200_ddpm_step(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr() if noise else None,
                                   d[3].data_ptr() if vm else None, C.byref(c), prev.data_ptr(), x0.data_ptr(), n,
                                   stream()))
        outs.append((prev.cpu(), x0.cpu()))
    (prev, x0), (p2, x2) = outs
    assert torch.equal(bits(p2), bits(prev)) and torch.equal(bits(x2), bits(x0))
    ratio_report("ddpm_step", name, check_region(name, prev, 0, n, rp))
    ratio_report("ddpm_step_x0", name, check_region(name, x0, 0, n, rx))


PNDM = [  # name, n_hist, pred, prev, eps_out
    ("n1_eps", 1, E.PRED_EPSILON, True, True),
    ("n2_v", 2, E.PRED_V, True, True),
    ("n3_eps_out_null", 3, E.PRED_EPSILON, True, False),
    ("n4_v_eps_out_null", 4, E.PRED_V, True, False),
    ("n4_prev_null_prk_accumulation", 4, E.PRED_EPSILON, False, True),
    ("n2_prev_null", 2, E.PRED_V, False, True),
]


@pytest.mark.parametrize("name,nh,pred,want_prev,want_eps", PNDM, ids=[c[0] for c in PNDM])
def test_pndm_step_matches_emulator(cuda_device, lib, name, nh, pred, want_prev, want_eps):
    n = 100_001
    g = gen(name)
    hist = [torch.randn(n, generator=g) for _ in range(nh)] + [torch.full((n,), NAN) for _ in range(4 - nh)]
    s = torch.randn(n, generator=g)
    w = {1: [1.0], 2: [1.5, -0.5], 3: [23 / 12, -16 / 12, 5 / 12], 4: [55 / 24, -59 / 24, 37 / 24, -9 / 24]}[nh]
    c = PndmCoef()
    for k in range(4):
        c.w[k] = w[k] if k < nh else NAN                     # slots >= n_hist: weight and history NaN, never read
    c.n_hist, c.sample_coeff, c.eps_coeff, c.v_alpha, c.v_beta, c.prediction_type = nh, 1.0123, 0.0456, 0.6, 0.8, pred
    cn = NS(w=[f32v(c.w[k]) for k in range(4)], n_hist=nh, sample_coeff=f32v(1.0123), eps_coeff=f32v(0.0456),
            v_alpha=f32v(0.6), v_beta=f32v(0.8), prediction_type=pred)
    rp, re = E.pndm_step(hist, s if want_prev else None, cn, n)
    hd = [h.cuda() for h in hist]
    hp = (C.c_void_p * 4)(*[h.data_ptr() for h in hd])
    sd = s.cuda()
    outs = []
    for _ in range(2):
        prev, eps = sentinel32(n + 5).cuda(), sentinel32(n + 5).cuda()
        sync_ok(lib.b200_pndm_step(hp, sd.data_ptr() if want_prev else None, C.byref(c),
                                   prev.data_ptr() if want_prev else None, eps.data_ptr() if want_eps else None, n,
                                   stream()))
        outs.append((prev.cpu(), eps.cpu()))
    (prev, eps), (p2, e2) = outs
    assert torch.equal(bits(p2), bits(prev)) and torch.equal(bits(e2), bits(eps))
    if want_prev:
        ratio_report("pndm_step", name, check_region(name, prev, 0, n, rp))
    else:
        assert torch.isnan(prev).all()
    if want_eps:
        ratio_report("pndm_step_eps", name, check_region(name, eps, 0, n, re))
    else:
        assert torch.isnan(eps).all()


@pytest.mark.parametrize("N,sign", [(1, 1.0), (2, -1.0), (3, 1.0), (3, -1.0)])
def test_add_noise_matches_emulator(cuda_device, lib, N, sign):
    per = 70_001
    g = gen(f"an{N}{sign}")
    x0, z = torch.randn(N * per, generator=g), torch.randn(N * per, generator=g)
    ca, cb = torch.rand(N, generator=g), torch.rand(N, generator=g)
    want = E.add_noise(x0, z, ca, cb, sign, N, per)
    d = [t.cuda() for t in (x0, z, ca, cb)]
    outs = []
    for _ in range(2):
        y = sentinel32(N * per + 11).cuda()
        sync_ok(lib.b200_add_noise(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), d[3].data_ptr(), sign, N, per,
                                   y.data_ptr(), stream()))
        outs.append(y.cpu())
    assert torch.equal(bits(outs[0]), bits(outs[1]))
    ratio_report("add_noise", f"N{N}_sign{int(sign)}", check_region("add_noise", outs[0], 0, N * per, want))


@pytest.mark.parametrize("n", [1, 4099, 1_000_003])
def test_small_fp32_helpers_match_emulator(cuda_device, lib, n):
    g = gen(f"f32h{n}")
    a, b, c = (3 * torch.randn(n, generator=g) for _ in range(3))
    d = [t.cuda() for t in (a, b, c)]
    for entry, call, want in (
        ("exp_half_clamped", lambda y: lib.b200_exp_half_clamped(d[0].data_ptr(), -5.0, 4.0, y.data_ptr(), n, stream()),
         E.exp_half_clamped(a, -5.0, 4.0, n)),
        ("fma_f32", lambda y: lib.b200_fma_f32(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), y.data_ptr(), n,
                                               stream()), E.fma_f32(a, b, c, n)),
        ("scale_f32", lambda y: lib.b200_scale_f32(d[0].data_ptr(), 0.18215, 3.0, y.data_ptr(), n, stream()),
         E.scale_f32(a, 0.18215, 3.0, n)),
    ):
        outs = []
        for _ in range(2):
            y = sentinel32(n + 7).cuda()
            sync_ok(call(y))
            outs.append(y.cpu())
        assert torch.equal(bits(outs[0]), bits(outs[1])), entry
        ratio_report(entry, f"n{n}", check_region(entry, outs[0], 0, n, want))


@pytest.mark.parametrize("n", [1, 1000, 100_003])
def test_vae_reparam_kld_matches_emulator(cuda_device, lib, n):
    g = gen(f"vae{n}")
    mu, lv, eps = torch.randn(n, generator=g), torch.randn(n, generator=g), torch.randn(n, generator=g)
    zw, kw = E.vae_reparam_kld(mu, lv, eps, n)
    d = [t.cuda() for t in (mu, lv, eps)]
    outs = []
    for _ in range(2):
        z, kld = sentinel32(n + 3).cuda(), sentinel32(2).cuda()
        sync_ok(lib.b200_vae_reparam_kld(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), z.data_ptr(),
                                         kld.data_ptr(), n, stream()))
        outs.append((z.cpu(), kld.cpu()))
    (z, kld), (z2, k2) = outs
    assert torch.equal(bits(z), bits(z2)) and torch.equal(bits(kld), bits(k2)), "the fixed-order KL sum must repeat"
    ratio_report("vae_reparam_kld_z", f"n{n}", check_region("z", z, 0, n, zw))
    ratio_report("vae_reparam_kld_kld", f"n{n}", check_region("kld", kld, 0, 1, kw))


# ------------------------------------------------------------------------------------------------------------------
# ddpm_kl
# ------------------------------------------------------------------------------------------------------------------
def kl_struct(is_t0, pred=E.PRED_EPSILON, clip=1):
    c = KlCoef()
    c.sqrt_alpha_prod_t, c.sqrt_beta_prod_t, c.coef_x0, c.coef_xt = 0.9, math.sqrt(1 - 0.81), 0.3, 0.65
    c.log_pred_var = math.log(1e-4) if is_t0 else math.log(0.02)
    c.log_post_var, c.bin_width = math.log(0.015), 2.0 / 255
    c.prediction_type, c.clip, c.is_t0 = pred, clip, is_t0
    return c


KL = [  # name, N, per_sample, is_t0, pred, clip
    ("kl_N3_per1000", 3, 1000, 0, E.PRED_EPSILON, 1),
    ("kl_N3_per100003_v", 3, 100_003, 0, E.PRED_V, 0),
    ("decoder_nll_N3_edges", 3, 5000, 1, E.PRED_EPSILON, 1),
    ("decoder_nll_N1_sample_pred", 1, 777, 1, E.PRED_SAMPLE, 0),
    ("kl_N1_c3_volume_160x224x160", 1, 160 * 224 * 160, 0, E.PRED_EPSILON, 1),
    ("decoder_nll_N1_c3_volume_160x224x160", 1, 160 * 224 * 160, 1, E.PRED_EPSILON, 1),
]


@pytest.mark.parametrize("name,N,per,is_t0,pred,clip", KL, ids=[c[0] for c in KL])
def test_ddpm_kl_matches_emulator(cuda_device, lib, name, N, per, is_t0, pred, clip):
    """kl_out against the emulator's bound; sample_sum against the float64 sum of the kernel's own kl_out, and against
    the emulator's sums within their bound.  Every term reaches sample_sum through at most L fp64 additions: its
    thread's ceil(per / threads) terms, the 5 + 3 levels of the warp and block trees and one atomic per CTA of the
    sample, so the fp64 sum is within L 2^-53 sum |kl| of the exact one.  A thread that sums its terms in fp32 is
    ~ sqrt(terms) 2^-24 off per partial: at the C3 volume (43 terms per thread) that is 10^4 times L 2^-53."""
    g = gen(name)
    a = (torch.rand(N * per, generator=g) * 2 - 1)
    edges = torch.tensor([0.999, -0.999], dtype=torch.float32)
    step = torch.nextafter(edges, torch.tensor([2.0, -2.0]))
    back = torch.nextafter(edges, torch.tensor([0.0, 0.0]))
    a[:6] = torch.cat([edges, step, back])                   # exactly at +-0.999f and one fp32 step either side
    s = 0.9 * a + 0.44 * torch.randn(N * per, generator=g)
    m = (s - 0.9 * a) / 0.44 + 0.05 * torch.randn(N * per, generator=g)
    c = kl_struct(is_t0, pred, clip)
    cn = NS(**{k: getattr(c, k) for k, _ in KlCoef._fields_})
    want, wsum, wsum_err = E.ddpm_kl(a, s, m, cn, N, per)
    d = [t.cuda() for t in (a, s, m)]
    outs = []
    for _ in range(2):
        kl = sentinel32(N * per + 13).cuda()
        ssum = torch.full((N + 1,), 0.5, dtype=torch.float64, device="cuda")
        sync_ok(lib.b200_ddpm_kl(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), C.byref(c), kl.data_ptr(),
                                 ssum.data_ptr(), N, per, stream()))
        outs.append((kl.cpu(), ssum.cpu()))
    (kl, ssum), (kl2, _) = outs
    assert torch.equal(bits(kl), bits(kl2))
    assert ssum[N] == 0.5, "stores past sample_sum[N - 1]"
    ratio_report("ddpm_kl", name, check_region(name, kl, 0, N * per, want))
    K = kl[:N * per].double().view(N, per)
    got = ssum[:N] - 0.5
    own = K.sum(1)
    ctas = min((per + 255) // 256, 4 * lib.b200_sm_count())
    L = -(-per // (ctas * 256)) + 8 + ctas
    tol = L * 2.0 ** -53 * (K.abs().sum(1) + 0.5) + 2.0 ** -52
    r = float(((got - own).abs() / tol).max())
    ratio_report("ddpm_kl_sample_sum", name, r)
    assert r <= 1, f"{name}: sample_sum {got.tolist()} vs the fp64 sum of kl_out {own.tolist()} (tol {tol.tolist()})"
    assert ((got - wsum).abs() <= wsum_err + tol).all()


# ------------------------------------------------------------------------------------------------------------------
# vq_argmin_gather
# ------------------------------------------------------------------------------------------------------------------
VQ = [  # name, M, D, K, ste, features ("dup": duplicated rows in lanes k, k+1, k+32; "nan": an all-NaN row)
    ("tiled_D32_M_mod4_0_K256", 256, 32, 256, 1, "dup"),
    ("tiled_D32_M_mod4_1_K256", 257, 32, 256, 0, "dup"),
    ("tiled_D32_M_mod4_2_K1024", 1026, 32, 1024, 1, ""),
    ("tiled_D32_M_mod4_3_K33_nan_row", 515, 32, 33, 1, "nan"),
    ("tiled_D32_M1_K2", 1, 32, 2, 0, ""),
    ("generic_D1_K2", 999, 1, 2, 1, ""),
    ("generic_D3_K33_dup", 1001, 3, 33, 0, "dup"),
    ("generic_D64_K700_near_the_shared_memory_limit", 700, 64, 700, 1, "dup"),
    ("generic_D64_K1_single_code", 50, 64, 1, 1, ""),
    ("generic_D3_K256_nan_row", 300, 3, 256, 0, "nan"),
]


@pytest.mark.parametrize("name,M,D,K,ste,feat", VQ, ids=[c[0] for c in VQ])
def test_vq_argmin_gather_matches_emulator(cuda_device, lib, name, M, D, K, ste, feat):
    g = gen(name)
    X = torch.randn(M, D, generator=g)
    cb = torch.randn(K, D, generator=g)
    if "dup" in feat and K > 40:
        k0 = 5
        for k in (k0, k0 + 1, k0 + 32):                     # three lanes hold the same code as row 0's input
            cb[k] = X[0]
        X[1] = cb[k0 + 32] + 1e-3
    if "nan" in feat:
        X[M // 2] = NAN
    xp, qp = D + 5, D + 11
    x = nan_rows(X, xp)
    want = E.vq_argmin_gather(x, M, D, xp, cb.reshape(-1), K, qp, ste)
    xd, cd = x.cuda(), cb.reshape(-1).cuda()
    results = []
    for _ in range(2):
        idx = torch.full((M + 4,), -7, dtype=torch.int64, device="cuda")
        q16 = sentinel16((M + 2) * qp).cuda()
        q32 = sentinel32((M + 2) * D).cuda()
        sq = torch.full((2,), 0.25, dtype=torch.float64, device="cuda")
        hist = torch.zeros(K + 3, dtype=torch.int32, device="cuda")
        sync_ok(lib.b200_vq_argmin_gather(xd.data_ptr(), M, D, xp, cd.data_ptr(), K, idx.data_ptr(), q16.data_ptr(), qp,
                                          q32.data_ptr(), ste, sq.data_ptr(), hist.data_ptr(), stream()))
        results.append([t.cpu() for t in (idx, q16, q32, sq, hist)])
    (idx, q16, q32, sq, hist), again = results
    for a_, b_ in zip((idx, q16, q32, hist), (again[0], again[1], again[2], again[4])):
        assert torch.equal(bits(a_), bits(b_)), f"{name}: repeats differ"
    assert (idx[M:] == -7).all() and (hist[K:] == 0).all(), f"{name}: stores past M rows / K codes"
    bad = torch.nonzero(idx[:M] != want.idx).flatten()
    if bad.numel():
        pytest.fail(f"{name}: {bad.numel()} indices differ, first at row {int(bad[0])}: got {int(idx[bad[0]])} want "
                    f"{int(want.idx[bad[0]])}; float64 gap to the runner-up there {float(want.gap[bad[0]]):.3g} (a gap "
                    f"within fp32 rounding of the distances is the emulator's own double rounding)")
    if "dup" in feat and K > 40:
        assert int(idx[0]) == 5, "ties must go to the lowest index"
    if "nan" in feat:
        assert int(idx[M // 2]) == 0, "an all-NaN row takes index 0"
    assert torch.equal(hist[:K].long(), want.hist), f"{name}: histogram differs"
    assert (bits(q16[M * qp:]) == SENT16).all() and torch.isnan(q32[M * D:]).all(), f"{name}: stores past M rows"
    assert torch.equal(bits(q16[:M * qp].view(M, qp)), bits(want.q16.to(H16))), f"{name}: q_h16 differs"
    q = q32[:M * D].view(M, D).double()
    same = (q == want.q32) | (torch.isnan(q) & torch.isnan(want.q32))
    assert same.all(), f"{name}: q_f32 differs"
    got_sq = float(sq[0]) - 0.25
    assert sq[1] == 0.25
    if math.isnan(want.sqerr):
        assert math.isnan(got_sq)
    else:
        assert abs(got_sq - want.sqerr) <= want.sqerr_err + 2.0 ** -52 * 0.25, (got_sq, want.sqerr)
    # the optional outputs on their own: indices only
    idx2 = torch.full((M + 4,), -7, dtype=torch.int64, device="cuda")
    sync_ok(lib.b200_vq_argmin_gather(xd.data_ptr(), M, D, xp, cd.data_ptr(), K, idx2.data_ptr(), None, 0, None, ste,
                                      None, None, stream()))
    assert torch.equal(idx2.cpu(), idx), f"{name}: indices depend on the optional outputs"

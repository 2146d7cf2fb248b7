"""b200_interpolate, b200_upsample2x_interp and b200_pool_s2 on the GPU against tests/resample_emulator.py, which
reproduces their fp32 sequences bit for bit.  Every case builds its operands as host tensors in the ABI layout, runs
the reading on them and the library on device copies, and checks:

  values       every stored element equal to the reading (NaN equal to NaN);
  footprint    the output buffer is prefilled with a NaN bit pattern, with a leading offset and a trailing margin; only
               the elements the header says are written change;
  ignored      input elements the call must not read (channels past round_up(C, 8) or past C, the gaps of a strided
               layout) hold NaN;
  determinism  a second identical call stores identical bits.

Argument checks run without a GPU in tests/test_elementwise_args_cpu.py.  Non-finite inputs pin the copied axes of the
linear family (inf stays inf) and the first even output of the bilinear x2 upsampling (an inf in row 0 stays inf).
"""
import math
import zlib

import pytest
import torch

from generativemodels_b200 import _lib, ops
from tests import elementwise_emulator as E
from tests import resample_emulator as R

pytestmark = pytest.mark.gpu

H16 = ops.H16
NAN = float("nan")
INF = float("inf")
DT_H16, DT_F32, DT_F64, DT_FP16, DT_BF16 = 0, 1, 2, 3, 4
TORCH_DT = {DT_H16: H16, DT_F32: torch.float32, DT_F64: torch.float64, DT_FP16: torch.float16,
            DT_BF16: torch.bfloat16}
MODES = {"nearest": R.NEAREST, "linear": R.LINEAR, "bilinear": R.BILINEAR, "bicubic": R.BICUBIC,
         "trilinear": R.TRILINEAR, "area": R.AREA}
MODE_DIMS = {"nearest": (1, 2, 3), "linear": (1,), "bilinear": (2,), "bicubic": (2,), "trilinear": (3,),
             "area": (1, 2, 3)}


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def bits(x):
    return x.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()])


@pytest.fixture(scope="module")
def lib():
    return _lib.require_device()


def sync_ok(rc):
    torch.cuda.synchronize()
    assert rc == 0, (rc, _lib.last_error())


def report(entry, name):
    print(f"\nBOUND {entry} {name} max(err/tol) = 0.000 (bit-exact)")


def same_values(name, want, got):
    ex = E.excess(want, got.to(torch.float64))
    if not (ex == 0).all():
        i = tuple(int(j) for j in torch.nonzero(ex != 0)[0])
        pytest.fail(f"{name}: got {float(got[i])} want {float(want.out[i])} at {i}; {int((ex != 0).sum())} of "
                    f"{ex.numel()} differ")


def span(shape, strides):
    return 1 + sum((s - 1) * st for s, st in zip(shape, strides))


def cl_strides(D, H, W, pitch):
    return (D * H * W * pitch, 1, H * W * pitch, W * pitch, pitch)


def planar_strides(C, D, H, W):
    return (C * D * H * W, D * H * W, H * W, W, 1)


def run_interpolate(lib, name, mode, dims, shape, out, xdt=DT_H16, ydt=DT_H16, xs=None, ys=None, x_off=8, y_off=8,
                    ratios=None, scale=1.0, special=None):
    """One b200_interpolate case; returns nothing, fails on any check.  shape (N, C, D, H, W), out (OD, OH, OW)."""
    N, C, D, H, W = shape
    OD, OH, OW = out
    xs = xs or planar_strides(C, D, H, W)
    ys = ys or planar_strides(C, OD, OH, OW)
    xt, yt = TORCH_DT[xdt], TORCH_DT[ydt]
    xe, ye = torch.empty(0, dtype=xt).element_size(), torch.empty(0, dtype=yt).element_size()
    vec = R.vector_path(C, xdt, xs, ys, x_off * xe, y_off * ye)
    Cw = (C + 7) // 8 * 8 if vec else C                      # channels read and written
    g = gen(name)
    xbuf = torch.full((x_off + span((N, Cw, D, H, W), xs) + 16,), NAN, dtype=torch.float32).to(xt)
    xv = torch.as_strided(xbuf, (N, Cw, D, H, W), xs, x_off)
    vals = scale * torch.randn(N, Cw, D, H, W, generator=g)
    if special is not None:
        special(vals)
    if xt is torch.float16:
        vals = vals.clamp(-65504, 65504)
    one = [1 if st == 0 else n for n, st in zip(xv.shape, xs)]     # a stride-0 axis holds one value
    torch.as_strided(xbuf, one, xs, x_off).copy_(vals[tuple(slice(0, n) for n in one)].to(xt))
    src = xv.clone()
    if ratios is None:
        ratios = [float(torch.tensor(i, dtype=torch.float32) / torch.tensor(o, dtype=torch.float32))
                  for i, o in zip((D, H, W), out)]
    want = R.interpolate(src, out[3 - dims:], ratios[3 - dims:], MODES[mode], ydt == DT_H16)
    ny = y_off + span((N, Cw, OD, OH, OW), ys) + 24
    xd = xbuf.cuda()
    xst, yst = (ctypes_i64(xs), ctypes_i64(ys))
    outs = []
    for _ in range(2):
        yd = torch.full((ny,), NAN, dtype=torch.float32).to(yt).cuda()
        rd, rh, rw = ratios
        rc = lib.b200_interpolate(xd.data_ptr() + x_off * xe, xdt, xst, yd.data_ptr() + y_off * ye, ydt, yst, N, C, D,
                                  H, W, OD, OH, OW, dims, MODES[mode], rd, rh, rw, ops._stream())
        sync_ok(rc)
        outs.append(yd.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y)), f"{name}: a second call stores different bits"
    got = torch.as_strided(y, (N, Cw, OD, OH, OW), ys, y_off)
    same_values(name, want, got)
    mask = torch.zeros(ny, dtype=torch.bool)
    torch.as_strided(mask, (N, Cw, OD, OH, OW), ys, y_off).fill_(True)
    assert torch.isnan(y[~mask].float()).all(), f"{name}: stores outside the output"
    report("interpolate", name)
    return got, vec


def ctypes_i64(v):
    import ctypes as C
    return (C.c_int64 * 5)(*v)


# ------------------------------------------------------------------------------------------------------------------
# interpolate: every mode x dims, both thread mappings, every input dtype, both output dtypes
# ------------------------------------------------------------------------------------------------------------------
def _extent(dims, spatial):
    return (1,) * (3 - dims) + spatial[3 - dims:]


MODE_CASES = []
for m, dd in MODE_DIMS.items():
    for d in dd:
        for sizes, tag in (((5, 7, 9), (3, 12, 4)), "odd_size"), (((4, 6, 8), (8, 3, 16)), "even"):
            MODE_CASES.append((m, d, sizes, tag))


@pytest.mark.parametrize("mode,dims,sizes,tag", MODE_CASES, ids=[f"{c[0]}_dims{c[1]}_{c[3]}" for c in MODE_CASES])
@pytest.mark.parametrize("layout", ["planar_f32_to_f32", "cl_h16_vec_C13", "cl_f32_vec_C8", "cl_h16_misaligned"])
def test_interpolate_modes_and_layouts(cuda_device, lib, mode, dims, sizes, tag, layout):
    (D, H, W), (OD, OH, OW) = sizes
    D, H, W = _extent(dims, (D, H, W))
    OD, OH, OW = _extent(dims, (OD, OH, OW))
    N = 2
    name = f"{mode}_{dims}_{tag}_{layout}"
    if layout == "planar_f32_to_f32":
        C = 3
        run_interpolate(lib, name, mode, dims, (N, C, D, H, W), (OD, OH, OW), DT_F32, DT_F32)
    elif layout == "cl_h16_vec_C13":
        C, xp, yp = 13, 24, 16
        _, vec = run_interpolate(lib, name, mode, dims, (N, C, D, H, W), (OD, OH, OW), DT_H16, DT_H16,
                                 cl_strides(D, H, W, xp), cl_strides(OD, OH, OW, yp))
        assert vec
    elif layout == "cl_f32_vec_C8":
        C, xp, yp = 8, 16, 8
        _, vec = run_interpolate(lib, name, mode, dims, (N, C, D, H, W), (OD, OH, OW), DT_F32, DT_H16,
                                 cl_strides(D, H, W, xp), cl_strides(OD, OH, OW, yp))
        assert vec
    else:
        C, xp, yp = 5, 8, 8
        _, vec = run_interpolate(lib, name, mode, dims, (N, C, D, H, W), (OD, OH, OW), DT_H16, DT_F32,
                                 cl_strides(D, H, W, xp), cl_strides(OD, OH, OW, yp), x_off=9)
        assert not vec


SCALAR = [  # name, x dtype, x strides builder, note
    ("permuted_strides_f64", DT_F64, lambda N, C, D, H, W: (C * D * H * W, 1, W * H * C, C, H * C)),
    ("broadcast_c_stride0_fp16", DT_FP16, lambda N, C, D, H, W: (D * H * W, 0, H * W, W, 1)),
    ("gapped_rows_bf16", DT_BF16, lambda N, C, D, H, W: (C * D * H * (W + 3) + 5, D * H * (W + 3), H * (W + 3), W + 3, 1)),
]


@pytest.mark.parametrize("mode", ["nearest", "bilinear", "bicubic", "area"])
@pytest.mark.parametrize("name,xdt,strides", SCALAR, ids=[c[0] for c in SCALAR])
def test_interpolate_scalar_path_dtypes_and_strides(cuda_device, lib, mode, name, xdt, strides):
    N, C, D, H, W, OH, OW = 2, 3, 1, 7, 6, 4, 11
    run_interpolate(lib, f"{name}_{mode}", mode, 2, (N, C, D, H, W), (1, OH, OW), xdt, DT_H16,
                    strides(N, C, D, H, W), x_off=3, y_off=5)


@pytest.mark.parametrize("mode", ["nearest", "bilinear", "bicubic"])
@pytest.mark.parametrize("n_in,factor", [(17, 0.5), (15, 0.5), (17, 1.5), (9, 2.5), (5, 1.1)])
def test_interpolate_scale_factor_against_size(cuda_device, lib, mode, n_in, factor):
    """The ratio F.interpolate forms from a scale factor, float(1 / scale_factor), differs from in / out on odd
    extents; both go through the kernel as the caller gives them."""
    n_out = int(math.floor(n_in * factor))
    for tag, r in (("scale", float(torch.tensor(1.0 / factor, dtype=torch.float32))),
                   ("size", float(torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)))):
        run_interpolate(lib, f"{mode}_{n_in}_{factor}_{tag}", mode, 2, (1, 2, 1, n_in, n_in + 2),
                        (1, n_out, n_out + 1), DT_F32, DT_F32, ratios=[1.0, r, r])


def _nonfinite(v):
    """inf, -inf and NaN at three voxels of every channel (the last H row when H == 1)."""
    h = min(v.shape[3] - 1, 1)
    v[..., 0, h, 2] = INF
    v[..., 0, h * 2, 0] = -INF
    v[..., 0, h * 3, 3] = NAN


@pytest.mark.parametrize("mode,dims", [("linear", 1), ("bilinear", 2), ("trilinear", 3), ("nearest", 2)])
@pytest.mark.parametrize("layout", ["planar_f32", "cl_h16_vec"])
def test_interpolate_identity_axes_copy_nonfinite(cuda_device, lib, mode, dims, layout):
    """An axis of the linear family with out == in is a copy: inf stays inf, NaN stays NaN (not inf * 0)."""
    D, H, W = _extent(dims, (3, 5, 6))
    out = _extent(dims, (3, 5, 6))
    if layout == "planar_f32":
        got, _ = run_interpolate(lib, f"identity_{mode}_{layout}", mode, dims, (1, 2, D, H, W), out, DT_F32, DT_F32,
                                 special=_nonfinite)
    else:
        got, _ = run_interpolate(lib, f"identity_{mode}_{layout}", mode, dims, (1, 8, D, H, W), out, DT_H16, DT_H16,
                                 cl_strides(D, H, W, 8), cl_strides(*out, 8), special=_nonfinite)
    if layout == "planar_f32" or H16 is torch.bfloat16:
        assert torch.isinf(got.float()).sum() == 2 * got.shape[1] and torch.isnan(got.float()).sum() == got.shape[1]


@pytest.mark.parametrize("mode", ["bilinear", "trilinear"])
def test_interpolate_partly_identity_keeps_inf_along_the_copied_axis(cuda_device, lib, mode):
    """Only W changes: each output row interpolates one input row, so an inf pollutes only its own row."""
    dims = 2 if mode == "bilinear" else 3
    D, H, W = _extent(dims, (2, 4, 5))
    OD, OH, OW = _extent(dims, (2, 4, 9))
    got, _ = run_interpolate(lib, f"partly_identity_{mode}", mode, dims, (1, 3, D, H, W), (OD, OH, OW), DT_F32,
                             DT_F32, special=lambda v: v[..., 0, 1, 2].fill_(INF))
    assert torch.isfinite(got[..., 0, 0, :]).all() and not torch.isfinite(got[..., 0, 1, :]).all()


@pytest.mark.parametrize("mode,n_in,n_out", [("linear", 1 << 24, 5), ("nearest", 5, 1 << 24), ("area", 1 << 16, 65535),
                                             ("area", 65535, 1 << 16)])
def test_interpolate_largest_extents(cuda_device, lib, mode, n_in, n_out):
    """Extents at the header's limits: 2^24 per axis; AREA at in * out + out = 2^32 - 1 and = 2^32."""
    run_interpolate(lib, f"{mode}_{n_in}_to_{n_out}", mode, 1, (1, 1, 1, 1, n_in), (1, 1, n_out), DT_F32, DT_F32)


@pytest.mark.parametrize("mode,n_in,n_out", [("linear", (1 << 24) + 1, 5), ("nearest", 5, (1 << 24) + 1),
                                             ("area", 6700416, 641), ("area", 640, 6700417)])
def test_interpolate_past_the_limits_is_einval(cuda_device, lib, mode, n_in, n_out):
    x = torch.zeros(64, device="cuda")
    st = ctypes_i64((1, 1, 1, 1, 0))
    rc = lib.b200_interpolate(x.data_ptr(), DT_F32, st, x.data_ptr(), DT_F32, st, 1, 1, 1, 1, n_in, 1, 1, n_out, 1,
                              MODES[mode], 1.0, 1.0, float(n_in) / n_out, ops._stream())
    assert rc == _lib.B200_EINVAL, (rc, _lib.last_error())


def test_interpolate_offsets_past_2pow31(cuda_device, lib):
    """N = 2 with batch strides past 2^31 elements on both sides (h16, 8-channel vectors)."""
    C, H, W, OH, OW = 8, 6, 5, 9, 3
    bs = (1 << 31) + 64
    xs, ys = (bs, 1, H * W * C, W * C, C), (bs, 1, OH * OW * C, OW * C, C)
    g = gen("past2pow31")
    vals = torch.randn(2, H, W, C, generator=g).to(H16)
    xd = torch.full((bs + H * W * C,), NAN, dtype=H16, device="cuda")
    for n in range(2):
        xd[n * bs:n * bs + H * W * C] = vals[n].reshape(-1).cuda()
    src = vals.permute(0, 3, 1, 2).unsqueeze(2)
    want = R.interpolate(src, (OH, OW), (float(torch.tensor(H / OH, dtype=torch.float32)),
                                         float(torch.tensor(W / OW, dtype=torch.float32))), R.BILINEAR, True)
    outs = []
    for _ in range(2):
        yd = torch.full((bs + OH * OW * C + 64,), NAN, dtype=H16, device="cuda")
        rc = lib.b200_interpolate(xd.data_ptr(), DT_H16, ctypes_i64(xs), yd.data_ptr(), DT_H16, ctypes_i64(ys), 2, C, 1,
                                  H, W, 1, OH, OW, 2, R.BILINEAR, 1.0, float(torch.tensor(H / OH, dtype=torch.float32)),
                                  float(torch.tensor(W / OW, dtype=torch.float32)), ops._stream())
        sync_ok(rc)
        assert int((~torch.isnan(yd)).sum()) == 2 * OH * OW * C, "stores outside the output"
        outs.append(torch.stack([yd[n * bs:n * bs + OH * OW * C].cpu() for n in range(2)]))
        del yd
    assert torch.equal(bits(outs[0]), bits(outs[1])), "a second call stores different bits"
    got = outs[0].view(2, OH, OW, C).permute(0, 3, 1, 2).unsqueeze(2)
    same_values("past2pow31", want, got)
    report("interpolate", "offsets_past_2pow31")


# ------------------------------------------------------------------------------------------------------------------
# upsample2x_interp (SPADENet)
# ------------------------------------------------------------------------------------------------------------------
def run_up2(lib, name, N, H, W, pitch, mode, C=None, scale=1.0, special=None):
    g = gen(name)
    X = torch.zeros(N, H, W, pitch)
    X[..., :C or pitch] = scale * torch.randn(N, H, W, C or pitch, generator=g)
    if special is not None:
        special(X)
    if H16 is torch.float16:
        X = X.clamp(-65504, 65504)
    x = torch.cat([X.reshape(-1).to(H16), torch.full((3 * pitch,), NAN).to(H16)])
    want = R.upsample2x_interp(x, N, H, W, pitch, mode)
    n = N * 4 * H * W * pitch
    xd = x.cuda()
    outs = []
    for _ in range(2):
        yd = torch.full((8 + n + 5 * pitch,), NAN).to(H16).cuda()
        sync_ok(lib.b200_upsample2x_interp(xd.data_ptr(), N, H, W, pitch, mode, yd[8:].data_ptr(), ops._stream()))
        outs.append(yd.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y)), f"{name}: a second call stores different bits"
    assert torch.isnan(y[:8].float()).all() and torch.isnan(y[8 + n:].float()).all(), f"{name}: footprint"
    got = y[8:8 + n].view(N, 2 * H, 2 * W, pitch)
    same_values(name, want, got)
    report("upsample2x_interp", name)
    return got


UP2 = [("N1_1x1", 1, 1, 1, 8), ("N2_1x2", 2, 1, 2, 8), ("N1_2x3", 1, 2, 3, 16), ("N3_3x1", 3, 3, 1, 8),
       ("N1_odd_7x5_pitch24", 1, 7, 5, 24), ("spadenet_8x8_C128", 1, 8, 8, 128), ("spadenet_16x16_C64", 2, 16, 16, 64),
       ("spadenet_32x32_C32", 1, 32, 32, 32)]


@pytest.mark.parametrize("mode", [_lib.INTERP_BILINEAR, _lib.INTERP_BICUBIC], ids=["bilinear", "bicubic"])
@pytest.mark.parametrize("name,N,H,W,pitch", UP2, ids=[c[0] for c in UP2])
def test_upsample2x_interp_bit_exact(cuda_device, lib, mode, name, N, H, W, pitch):
    run_up2(lib, f"{name}_{mode}", N, H, W, pitch, mode, C=max(pitch - 3, 1))


def test_upsample2x_bicubic_overshoot_saturates(cuda_device, lib):
    """A step of +-6e4 makes the Keys kernel overshoot past 65504; fp16 stores saturate there."""
    def step(X):
        X[:, :, :3] = 6e4
        X[:, :, 3:] = -6e4
    got = run_up2(lib, "bicubic_overshoot", 1, 4, 6, 8, _lib.INTERP_BICUBIC, special=step)
    if H16 is torch.float16:
        assert float(got.float().abs().max()) == 65504.0 and torch.isfinite(got.float()).all()


@pytest.mark.parametrize("mode", [_lib.INTERP_BILINEAR, _lib.INTERP_BICUBIC], ids=["bilinear", "bicubic"])
def test_upsample2x_border_inf(cuda_device, lib, mode):
    """inf in row 0 / column 0 (and NaN inside): bilinear's first even output weights row 1 by 0 and row 0 by 1, so
    the inf stays inf there, as ATen's does."""
    def spec(X):
        X[0, 0, 2, 0] = INF
        X[0, 3, 0, 1] = -INF
        X[0, 2, 2, 2] = NAN
    got = run_up2(lib, f"border_inf_{mode}", 1, 5, 4, 8, mode, special=spec)
    if mode == _lib.INTERP_BILINEAR and H16 is torch.bfloat16:
        assert got[0, 0, 4, 0].float() == INF and got[0, 6, 0, 1].float() == -INF


# ------------------------------------------------------------------------------------------------------------------
# pool_s2 (PatchGAN pyramid)
# ------------------------------------------------------------------------------------------------------------------
def run_pool(lib, name, N, D, H, W, pitch, dims, k, pad, mode, C=None, special=None):
    g = gen(name)
    X = torch.zeros(N, D, H, W, pitch)
    X[..., :C or pitch] = torch.randn(N, D, H, W, C or pitch, generator=g)
    if special is not None:
        special(X)
    x = torch.cat([X.reshape(-1).to(H16), torch.full((2 * pitch,), NAN).to(H16)])
    want = R.pool_s2(x, N, D, H, W, pitch, dims, k, pad, mode)
    n = want.out.numel()
    xd = x.cuda()
    outs = []
    for _ in range(2):
        yd = torch.full((8 + n + 3 * pitch,), NAN).to(H16).cuda()
        sync_ok(lib.b200_pool_s2(xd.data_ptr(), N, D, H, W, pitch, dims, k, pad, mode, yd[8:].data_ptr(),
                                 ops._stream()))
        outs.append(yd.cpu())
    y = outs[0]
    assert torch.equal(bits(outs[1]), bits(y)), f"{name}: a second call stores different bits"
    assert torch.isnan(y[:8].float()).all() and torch.isnan(y[8 + n:].float()).all(), f"{name}: footprint"
    got = y[8:8 + n].view(want.out.shape)
    same_values(name, want, got)
    if C is not None and special is None:
        assert (got[..., C:].float() == 0).all(), f"{name}: pad channels must stay zero"
    report("pool_s2", name)
    return got


POOL_KP = [(k, p) for k in range(1, 6) for p in range(k // 2 + 1)]


@pytest.mark.parametrize("mode", [_lib.POOL_AVG, _lib.POOL_MAX], ids=["avg", "max"])
@pytest.mark.parametrize("dims", [2, 3])
@pytest.mark.parametrize("k,pad", POOL_KP, ids=[f"k{k}p{p}" for k, p in POOL_KP])
def test_pool_s2_every_kernel_and_padding(cuda_device, lib, mode, dims, k, pad):
    N, D, H, W = (3, 2, 7, 9) if dims == 2 else (2, 6, 5, 8)
    run_pool(lib, f"k{k}p{pad}_dims{dims}_{mode}", N, D, H, W, 16, dims, k, pad, mode, C=11)


PATCHGAN = [("pyramid_64x64_C3", 1, 1, 64, 64, 8, 2), ("pyramid_32x32_C3", 1, 1, 32, 32, 8, 2),
            ("pyramid_3d_32cube", 1, 32, 32, 32, 8, 3), ("pyramid_3d_16x16x17", 2, 16, 16, 17, 8, 3)]


@pytest.mark.parametrize("mode", [_lib.POOL_AVG, _lib.POOL_MAX], ids=["avg", "max"])
@pytest.mark.parametrize("name,N,D,H,W,pitch,dims", PATCHGAN, ids=[c[0] for c in PATCHGAN])
def test_pool_s2_patchgan_pyramid(cuda_device, lib, mode, name, N, D, H, W, pitch, dims):
    run_pool(lib, f"{name}_{mode}", N, D, H, W, pitch, dims, 3, 1, mode, C=3)


@pytest.mark.parametrize("mode", [_lib.POOL_AVG, _lib.POOL_MAX], ids=["avg", "max"])
def test_pool_s2_nonfinite(cuda_device, lib, mode):
    def spec(X):
        X[0, 0, 1, 1, 0] = INF
        X[0, 0, 4, 2, 1] = -INF
        X[0, 0, 3, 5, 2] = NAN
        X[0, 0, 2, 2, 3] = NAN
        X[0, 0, 2, 3, 3] = INF
    run_pool(lib, f"nonfinite_{mode}", 1, 1, 7, 8, 8, 2, 3, 1, mode, special=spec)

"""SpatialRescaler and b200_interpolate on the H100: every case of the reference fixture (tests/golden/g_spatial_rescaler.pt);
a kernel sweep against F.interpolate over every mode and the dims it takes, down / up / identity / non-integer factors,
size versus scale factor, planar fp32, channels-last fp32 and channels-last h16 (and channels-last fp32 in, planar
out, the module's last stage), and 1 to 64 channels; B200_EINVAL for invalid calls; repeat calls and CUDA-graph replays
bit for bit.

F.interpolate is evaluated on the CPU, in fp32: the reference (and its fixture) run there, and ATen's CUDA kernels differ
from its CPU kernels in when they take copy shortcuts.  The sweep avoids the one CPU shortcut b200_interpolate does not
follow (tests/test_spatial_rescaler_cpu.py, _cpu_nearest2d_shortcut)."""
import ctypes as C
import itertools

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import _lib, ops
from generativemodels_b200.cuda_graph import graphed
from generativemodels_b200.networks.blocks import SpatialRescaler
from tests import rescaler_oracle as RO
from tests.golden import load

pytestmark = pytest.mark.gpu

GOLD = load("g_spatial_rescaler")
_MODE_DIMS = [("nearest", 1), ("nearest", 2), ("nearest", 3), ("linear", 1), ("bilinear", 2), ("bicubic", 2),
              ("trilinear", 3), ("area", 1), ("area", 2), ("area", 3)]
_LAYOUTS = ["planar", "cl_f32", "cl_h16", "cl_f32_to_planar"]
_CHANNELS = (1, 3, 8, 13, 64)
_ARGS = [dict(scale_factor=0.5), dict(scale_factor=2.0), dict(scale_factor=1.0), dict(scale_factor=1.7),
         dict(scale_factor=0.6), "odd_size"]
_EPS16 = 2.0 ** -10 if ops.H16 is torch.float16 else 2.0 ** -7


def _rescaler(kw, seed=0):
    return RO.seeded_weights(SpatialRescaler(**kw), seed).eval().cuda()


# ---- the module against the reference fixture -----------------------------------------------------------------------
@pytest.mark.parametrize("name", list(GOLD))
def test_fixture_case(cuda_device, name):
    g = GOLD[name]
    m = _rescaler(g["kwargs"])
    with torch.no_grad():
        got = m(RO.input_of(g).cuda()).cpu()
    want = g["out"]
    assert got.shape == want.shape and got.dtype == torch.float32
    if m.remap_output:
        rel = ((got - want).norm() / want.norm()).item()
        mx = ((got - want).abs().max() / want.abs().max()).item()
        assert rel < 2e-2 and mx < 4e-2, f"rel L2 {rel:.3e}, normalised max-abs {mx:.3e}"
    elif g["kwargs"].get("method") == "nearest":
        assert torch.equal(got, want)
    else:
        err = (got - want).abs().max().item()
        assert err <= RO.ulps_of(want, 16), f"max-abs {err:.3e} vs 16 ulps of max|out| {RO.ulps_of(want, 16):.3e}"


def test_caller_dtype(cuda_device):
    g = GOLD["size_mapper_bias"]
    m = _rescaler(g["kwargs"])
    x = RO.input_of(g).cuda()
    with torch.no_grad():
        for dt in (torch.float16, torch.bfloat16, torch.float64):
            y = m(x.to(dt))
            assert y.dtype == dt
            assert ((y.double().cpu() - g["out"].double()).norm() / g["out"].norm()) < 2e-2
        y = SpatialRescaler(multiplier=0.5, method="nearest")(x.half())
        assert y.dtype == torch.float16 and torch.equal(y, F.interpolate(x.half(), scale_factor=0.5))


# ---- the kernel against F.interpolate -------------------------------------------------------------------------------
def _to_cl(x, dtype, sd):
    """[N, C, *spatial] -> CL with storage ``dtype`` (pitch round_up(C, 8) for h16, round_up(C, 4) for fp32)."""
    N, C_ = x.shape[:2]
    spatial = (1,) * (3 - sd) + tuple(x.shape[2:])
    P = ops.round_up(C_, 8 if dtype == ops.H16 else 4)
    t = torch.zeros((N, *spatial, P), dtype=dtype, device="cuda")
    t[..., :C_] = x.reshape(N, C_, *spatial).movedim(1, -1).to(dtype)
    return ops.CL(t, C_, sd)


def _from_cl(a, sd):
    return a.t[..., :a.C].movedim(-1, 1).float().reshape(a.N, a.C, *a.t.shape[4 - sd:4])


def _run(x, arg, mode, layout):
    sd = x.dim() - 2
    if layout == "planar":
        return ops.interpolate(x, mode=mode, **arg)
    if layout == "cl_f32_to_planar":
        return ops.interpolate(_to_cl(x, torch.float32, sd), mode=mode, planar_out=True, **arg)
    dt = torch.float32 if layout == "cl_f32" else ops.H16
    y = ops.interpolate(_to_cl(x, dt, sd), mode=mode, **arg)
    assert y.t.dtype == dt and y.spatial_dims == sd
    return _from_cl(y, sd)


@pytest.mark.parametrize("layout", _LAYOUTS)
@pytest.mark.parametrize("mode,dims", _MODE_DIMS)
def test_kernel_vs_interpolate(cuda_device, mode, dims, layout):
    gen = torch.Generator().manual_seed(dims * 7 + _LAYOUTS.index(layout))
    ext = (9, 17, 7)[3 - dims:]
    h16 = layout == "cl_h16"
    for C_, arg in itertools.product(_CHANNELS, _ARGS):
        if arg == "odd_size":
            arg = dict(size=tuple(max(1, e // 2 + (e % 3)) for e in ext))
        x = torch.randn((2, C_, *ext), generator=gen)
        if h16:
            x = x.to(ops.H16).float()
        want = F.interpolate(x, mode=mode, **arg)
        got = _run(x.cuda(), arg, mode, layout).cpu()
        what = f"{mode} {dims}-D {layout} C={C_} {arg}"
        assert got.shape == want.shape, what
        if mode == "nearest":
            assert torch.equal(got, want), what
            continue
        tol = RO.ulps_of(x, 16)
        if h16:
            want = want.to(ops.H16).float()
            tol = tol + _EPS16 * want.abs()
        assert ((got - want).abs() <= tol).all(), f"{what}: max-abs {(got - want).abs().max().item():.3e}"


def test_nearest_follows_the_formula(cuda_device):
    # scale_factor=1.1 on 5 samples src 0, 0, 1, 2, 3 along every axis: min(floor(dst / 1.1), 4), no identity shortcut
    for dims in (1, 2, 3):
        x = torch.arange(5.0, device="cuda").view((1, 1) + (1,) * (dims - 1) + (5,)).expand((1, 1) + (5,) * dims)
        y = ops.interpolate(x, scale_factor=1.1, mode="nearest")
        assert y[(0, 0) + (0,) * (dims - 1)].tolist() == [0, 0, 1, 2, 3]


def test_vector_path_writes_pad_channels_from_the_input(cuda_device):
    x = torch.randn(1, 13, 6, 10, device="cuda")
    a = _to_cl(x, ops.H16, 2)
    y = ops.interpolate(a, scale_factor=1.5, mode="bilinear")
    assert y.t.shape[-1] == 16 and torch.equal(y.t[..., 13:], torch.zeros_like(y.t[..., 13:]))


# ---- argument checks ------------------------------------------------------------------------------------------------
def _call(lib, x, y, mode, dims, ext_in, ext_out, ratios=(1.0, 1.0, 0.5), xs=None, dt=_lib.DT_F32, ydt=None):
    st = (C.c_int64 * 5)(*(xs or (64, 16, 16, 16, 1)))
    return lib.b200_interpolate(x, dt, st, y, dt if ydt is None else ydt, (C.c_int64 * 5)(64, 16, 16, 16, 1), 1, 1,
                                *ext_in, *ext_out, dims, mode, *ratios, ops._stream())


def test_einval(cuda_device):
    lib = _lib.require_device()
    x = torch.zeros(4096, device="cuda")
    y = torch.zeros(4096, device="cuda")
    xp, yp = x.data_ptr(), y.data_ptr()
    ok = _call(lib, xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 8), (1, 1, 4))
    assert ok == _lib.B200_OK
    bad = [
        (xp, yp, _lib.INTERPOLATE_BILINEAR, 1, (1, 1, 8), (1, 1, 4)),           # mode / dims mismatch
        (xp, yp, _lib.INTERPOLATE_LINEAR, 2, (1, 8, 8), (1, 4, 4)),
        (xp, yp, _lib.INTERPOLATE_BICUBIC, 3, (8, 8, 8), (4, 4, 4)),
        (xp, yp, _lib.INTERPOLATE_TRILINEAR, 2, (1, 8, 8), (1, 4, 4)),
        (xp, yp, _lib.INTERPOLATE_NEAREST, 4, (1, 8, 8), (1, 4, 4)),
        (xp, yp, _lib.INTERPOLATE_NEAREST, 0, (1, 1, 1), (1, 1, 1)),
        (xp, yp, 6, 2, (1, 8, 8), (1, 4, 4)),                                   # unknown mode
        (xp, yp, -1, 2, (1, 8, 8), (1, 4, 4)),
        (xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 0), (1, 1, 4)),             # empty extents
        (xp, yp, _lib.INTERPOLATE_AREA, 1, (1, 1, 8), (1, 1, 0)),
        (xp, yp, _lib.INTERPOLATE_BILINEAR, 2, (2, 8, 8), (2, 4, 4)),           # D must be 1 for dims 2
        (xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 2, 8), (1, 2, 4)),             # H must be 1 for dims 1
        (None, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 8), (1, 1, 4)),           # null pointer
    ]
    for args in bad:
        assert _call(lib, *args) == _lib.B200_EINVAL, args
    assert _call(lib, xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 8), (1, 1, 4), ratios=(1.0, 1.0, 0.0)) == _lib.B200_EINVAL
    assert _call(lib, xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 8), (1, 1, 4), xs=(64, 16, 16, 16, -1)) == \
        _lib.B200_EINVAL
    assert _call(lib, xp, yp, _lib.INTERPOLATE_LINEAR, 1, (1, 1, 8), (1, 1, 4), dt=2) == _lib.B200_EINVAL
    # fp64 / fp16 / bf16 inputs are read on the scalar path; the output stays h16 or fp32
    for dt in (_lib.DT_F64, _lib.DT_FP16, _lib.DT_BF16):
        assert _call(lib, xp, yp, _lib.INTERPOLATE_AREA, 1, (1, 1, 8), (1, 1, 4), dt=dt, ydt=_lib.DT_F32) == _lib.B200_OK
        assert _call(lib, xp, yp, _lib.INTERPOLATE_AREA, 1, (1, 1, 8), (1, 1, 4), dt=_lib.DT_F32, ydt=dt) == \
            _lib.B200_EINVAL
    assert _call(lib, xp, yp, _lib.INTERPOLATE_AREA, 1, (1, 1, 8), (1, 1, 4), dt=5, ydt=_lib.DT_F32) == _lib.B200_EINVAL
    torch.cuda.synchronize()


# ---- determinism and graphs -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["stages_3", "mult_0_6_1_3", "bicubic_down", "area_up", "linear1d_mapper"])
def test_repeat_and_graph_replay_bit_identical(cuda_device, name):
    g = GOLD[name]
    m = _rescaler(g["kwargs"])
    x = RO.input_of(g).cuda()
    with torch.no_grad():
        a, b = m(x), m(x)
        gd = graphed(m)
        first, second = gd(x), gd(x)
    assert torch.equal(a, b) and torch.equal(a, first) and torch.equal(a, second)

"""The 128 x 256 two-CTA convolution kernel (b200_igemm impl = 3) against the 128-column kernel (impl = 2) and the
CUDA-core cross-check kernel (impl = 1): outputs, GroupNorm partials, and which kernel the planner says ran."""
import ctypes as C
import math

import pytest
import torch

from generativemodels_b200 import _lib, ops

pytestmark = pytest.mark.gpu


def within_one_ulp(a, b):
    """|a - b| <= one 16-bit ulp of the larger magnitude, elementwise."""
    a, b = a.float(), b.float()
    mant = 7 if ops.H16 == torch.bfloat16 else 10
    emin = -126 if ops.H16 == torch.bfloat16 else -14
    m = torch.maximum(a.abs(), b.abs()).clamp_min(2.0 ** emin)
    ulp = torch.exp2(torch.floor(torch.log2(m)) - mant)
    return bool(((a - b).abs() <= ulp).all())


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture
def plans(monkeypatch):
    """Record b200_igemm_plan's (column tile, splits, work items) for every implicit-GEMM launch."""
    seen = []
    raw = ops.igemm_raw
    lib = _lib.load()
    nsm = int(lib.b200_sm_count())

    def spy(p):
        out = (C.c_int32 * 4)()
        assert lib.b200_igemm_plan(C.byref(p), nsm, 0, out) == 0
        seen.append((p.impl, tuple(out)[:3]))
        raw(p)

    monkeypatch.setattr(ops, "igemm_raw", spy)
    monkeypatch.setattr(ops, "_GN_FUSE_MIN_ROWS", 1)
    return seen


def check_partials(out):
    t = out.t.float().cpu()[..., :out.C]
    gw = out.C // out.gn.shape[2]
    g = t.reshape(t.shape[0], -1, out.C // gw, gw).double()
    want = torch.stack([g.sum((1, 3)), (g * g).sum((1, 3))], -1)
    got = out.gn.double().sum(1).cpu()
    err = ((got - want).abs() / (want.abs() + 1.0)).max().item()
    assert err < 2e-4, err


def run3(fn):
    """fn(impl) -> CL for impl 3, 2, 1; the wide output must match the 128-column one to one ulp and the check kernel to
    1e-2, and its GroupNorm partials must describe what it stored."""
    o3, o2, o1 = fn(3), fn(2), fn(1)
    assert within_one_ulp(o3.t[..., :o3.C], o2.t[..., :o2.C]), rel_l2(o3.t, o2.t)
    assert rel_l2(o3.t[..., :o3.C], o1.t[..., :o1.C]) < 1e-2
    if o3.gn is not None:
        check_partials(o3)
        g3, g2 = o3.gn.double().sum(1), o2.gn.double().sum(1)
        assert (((g3 - g2).abs() / (g2.abs() + 1.0)).max().item()) < 2e-4
    return o3


def packed(cout, cin, k=3, stride=1, splits=None, sd=3):
    w = torch.randn(cout, cin, *([k] * sd)) / math.sqrt(cin * k ** sd)
    return ops.PackedConv(w.cuda(), torch.randn(cout).cuda(), stride, 1, splits=splits)


CASES = [
    # (name, N, cin splits, cout, spatial, stride, rowvec, residual, act1, scale, act2)
    ("c256_rowvec_n2_ragged", 2, [64], 256, (9, 20, 17), 1, True, False, ops.ACT_NONE, 1.0, ops.ACT_NONE),
    ("c512_more_units_than_clusters", 1, [128], 512, (16, 32, 40), 1, False, False, ops.ACT_NONE, 1.0, ops.ACT_NONE),
    ("c256_concat_residual_silu", 2, [64, 128], 256, (6, 10, 12), 1, True, True, ops.ACT_SILU, 0.5, ops.ACT_SILU),
    ("c256_stride2", 1, [64], 256, (17, 30, 33), 2, False, False, ops.ACT_NONE, 1.0, ops.ACT_NONE),
    ("c512_residual_scale", 2, [64], 512, (8, 12, 20), 1, True, True, ops.ACT_NONE, 2.0, ops.ACT_NONE),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_wide_conv_matches(cuda_device, plans, case):
    name, N, splits, cout, sp, stride, use_rv, use_res, act1, scale, act2 = case
    torch.manual_seed(len(name))
    xs = [ops.to_cl(torch.randn(N, c, *sp).cuda()) for c in splits]
    pc = packed(cout, sum(splits), stride=stride, splits=splits)
    od = pc.out_dims(*sp)
    rv = torch.randn(N, cout).cuda() if use_rv else None
    res = ops.to_cl(torch.randn(N, cout, *od).cuda()) if use_res else None
    out = run3(lambda impl: ops.conv(xs, pc, rowvec=rv, act1=act1, scale=scale, residual=res, act2=act2, impl=impl))
    assert out.gn is not None
    assert [pl[0] for impl, pl in plans if impl == 3] == [256]
    assert [pl[0] <= 128 for impl, pl in plans if impl == 2] == [True]


def test_wide_odd_m_tiles(cuda_device, plans):
    """5 M tiles of 128 x 1 x 1 (2-D 5 x 128 output): the last pair's partner runs the protocol on a clamped tile but
    stores nothing and adds nothing to the GroupNorm partials."""
    torch.manual_seed(5)
    x = ops.to_cl(torch.randn(1, 64, 5, 128).cuda())
    pc = packed(256, 64, sd=2)
    out = run3(lambda impl: ops.conv(x, pc, impl=impl))
    wide = [pl for impl, pl in plans if impl == 3]
    assert wide == [(256, 1, 3)]
    check_partials(out)


def test_wide_upsample_phases(cuda_device, plans):
    """The 8-phase upsample convolution: every phase writes every other voxel of the output (doubled strides), with
    per-phase GroupNorm slots."""
    torch.manual_seed(8)
    x = ops.to_cl(torch.randn(2, 256, 5, 9, 7).cuda())
    pu = ops.PackedUpsampleConv((torch.randn(256, 256, 3, 3, 3) / 80).cuda(), torch.randn(256).cuda())
    run3(lambda impl: ops.conv_upsample2x(x, pu, impl=impl))
    assert [pl[0] for impl, pl in plans if impl == 3] == [256] * 8


def test_wide_rejects_calls_outside_its_envelope(cuda_device):
    x = ops.to_cl(torch.randn(1, 64, 4, 6, 8).cuda())
    with pytest.raises(RuntimeError):
        ops.conv(x, packed(384, 64), impl=3)         # cout not a multiple of 256
    with pytest.raises(RuntimeError):
        ops.conv(x, packed(256, 64), out_f32=True, impl=3)

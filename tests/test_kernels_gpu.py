"""Op-level parity of every CUDA kernel (called through the C-ABI) against plain fp32 CPU arithmetic.

The checker for one op is the reference's own arithmetic: torch CPU fp32 functional ops (what the reference
executes on CPU, SURVEY.md §8c) applied to the SAME 16-bit-rounded inputs the kernel sees.  Tolerances: the
kernels take 16-bit operands (fp16 by default, bf16 in the second flavour) and accumulate in fp32, so a result differs
from the fp32 checker only by the final 16-bit rounding of the output (rel 2^-8 for bf16) plus accumulation-order noise -> atol/rtol 2e-2 on O(1) data; fp32-out
paths are held to 2e-3; integer outputs (VQ indices) are exact outside fp32 near-ties.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from generativemodels_b200 import ops

pytestmark = pytest.mark.gpu


def bf(x):
    return x.to(ops.H16).float()


def rel_err(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item(), (a - b).abs().max().item()


def assert_close(a, b, tol, what):
    r, m = rel_err(a, b)
    scale = b.float().abs().max().item() + 1e-6
    assert r < tol and m < 4 * tol * scale + 1e-5, f"{what}: rel-L2 {r:.3e}, max-abs {m:.3e} (scale {scale:.3e})"


def _ops():
    from generativemodels_b200 import ops
    return ops


def to_cl_ref(x):
    """NC[D]HW fp32 (cpu) -> CL on cuda via the library's own layout kernel."""
    ops = _ops()
    return ops.to_cl(x.cuda())


# ------------------------------------------------------------------------------------------------ layout
@pytest.mark.parametrize("shape", [(2, 3, 9, 7), (1, 1, 5, 6, 7), (2, 40, 4, 4, 5), (1, 256, 16, 16)])
def test_layout_roundtrip(cuda_device, shape):
    ops = _ops()
    x = torch.randn(shape)
    a = ops.to_cl(x.cuda())
    sd = len(shape) - 2
    ref = bf(x).movedim(1, -1)
    if sd == 2:
        ref = ref.unsqueeze(1)
    got = a.t[..., : shape[1]].float().cpu()
    assert torch.equal(got, ref)
    assert a.t[..., shape[1]:].abs().sum().item() == 0
    back = ops.from_cl(a).cpu()
    assert torch.equal(back, bf(x))


# ------------------------------------------------------------------------------------------------ igemm / conv
CONV_CASES = [
    # (spatial_dims, N, Cin, Cout, in_spatial, k, stride, padding)
    (2, 1, 64, 64, (16, 16), 3, 1, 1),
    (2, 2, 128, 256, (33, 17), 3, 1, 1),
    (2, 1, 96, 48, (20, 12), 3, 1, 1),
    (2, 2, 3, 32, (16, 16), 3, 1, 1),
    (2, 1, 32, 3, (16, 16), 3, 1, 1),
    (2, 1, 64, 64, (8, 8), 1, 1, 0),
    (2, 1, 512, 512, (16, 16), 3, 1, 1),
    (3, 1, 64, 64, (8, 8, 8), 3, 1, 1),
    (3, 1, 96, 160, (9, 20, 12), 3, 1, 1),
    (3, 2, 1, 32, (6, 10, 12), 3, 1, 1),
    (3, 1, 32, 1, (6, 10, 12), 3, 1, 1),
    (3, 1, 256, 256, (8, 16, 16), 3, 1, 1),
    (2, 1, 64, 64, (16, 16), 3, 2, 1),
    (2, 1, 128, 128, (17, 31), 3, 2, 1),
    (3, 1, 64, 96, (8, 12, 16), 3, 2, 1),
    (3, 1, 32, 64, (8, 8, 8), 4, 2, 1),
    (2, 1, 8, 8, (4, 4), 3, 1, 1),
    (3, 1, 8, 16, (4, 4, 4), 3, 1, 1),
    # grids of at least one tile per SM (several tiles per persistent CTA), wide outputs split into 128-column tiles,
    # even and odd tile counts, stride 2, two samples
    (2, 1, 64, 256, (160, 128), 3, 1, 1),
    (2, 1, 96, 256, (151, 129), 3, 1, 1),
    (2, 2, 64, 128, (104, 128), 3, 1, 1),
    (3, 1, 64, 512, (12, 40, 40), 3, 1, 1),
    (2, 1, 64, 256, (300, 260), 3, 2, 1),
    (2, 1, 64, 384, (100, 128), 1, 1, 0),
]


# Test ids of the implementation parameter: "tcgen05" is the stable id of impl = 0, the tensor-core kernel (now wgmma on
# sm_90a); the id is kept so that these tests keep their names across kernel generations.
IMPL_IDS = {0: "tcgen05", 1: "check"}


def _case_id(c):
    sd, N, Cin, Cout, sp, k, s, p = c
    return f"conv{sd}d_n{N}_{Cin}to{Cout}_" + "x".join(map(str, sp)) + f"_k{k}s{s}p{p}"


@pytest.mark.parametrize("impl", [1, 0], ids=IMPL_IDS.get)
@pytest.mark.parametrize("case", CONV_CASES, ids=[_case_id(c) for c in CONV_CASES])
def test_conv(cuda_device, case, impl):
    ops = _ops()
    sd, N, Cin, Cout, sp, k, s, p = case
    torch.manual_seed(hash(case) % 1000)
    x = torch.randn(N, Cin, *sp)
    w = torch.randn(Cout, Cin, *([k] * sd)) / math.sqrt(Cin * k ** sd)
    b = torch.randn(Cout)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(bf(x), bf(w), b, stride=s, padding=p)
    pc = ops.PackedConv(w.cuda(), b.cuda(), s, p)
    out = ops.conv(ops.to_cl(x.cuda()), pc, impl=impl)
    got = ops.from_cl(out)
    assert tuple(got.shape) == tuple(ref.shape)
    assert_close(got, ref, 1e-2, f"conv {case} impl={impl}")


@pytest.mark.parametrize("sd,N,Cin,Cout,sp,s", [
    (3, 1, 1, 256, (40, 36, 44), 1), (2, 2, 3, 64, (200, 190), 1), (3, 2, 2, 32, (65, 60, 81), 2),
    (3, 1, 256, 1, (40, 36, 44), 1), (2, 2, 128, 3, (200, 190), 1), (3, 1, 64, 4, (20, 30, 61), 1),
])
def test_conv_tap_reformulations(cuda_device, sd, N, Cin, Cout, sp, s):
    """Degenerate ends of the UNet above the row threshold: conv_in-like layers go through b200_tap_gather + a
    one-chunk GEMM, out-conv-like layers through a 1x1 GEMM (taps as columns) + b200_tap_sum; compared with F.conv
    and with the plain 27-tap implicit GEMM (the CUDA-core cross-check implementation, impl=1)."""
    ops = _ops()
    torch.manual_seed(13)
    x = torch.randn(N, Cin, *sp)
    w = torch.randn(Cout, Cin, *([3] * sd)) / math.sqrt(Cin * 3 ** sd)
    b = torch.randn(Cout)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(bf(x), bf(w), b, stride=s, padding=1)
    pc = ops.PackedConv(w.cuda(), b.cuda(), s, 1)
    assert (pc.tap_in is not None) != (pc.tap_out is not None)
    xc = ops.to_cl(x.cuda())
    rows = ref.numel() // Cout
    assert rows >= ops._TAP_MIN_ROWS
    got = ops.from_cl(ops.conv(xc, pc))
    assert tuple(got.shape) == tuple(ref.shape)
    assert_close(got, ref, 1e-2, "tap-reformulated conv vs F.conv")
    plain = ops.from_cl(ops.conv(xc, pc, impl=1))
    assert_close(got, plain, 1e-2, "tap-reformulated conv vs plain implicit GEMM")
    if pc.tap_out is not None:
        o32 = ops.conv(xc, pc, out_f32=True)
        assert_close(ops.from_cl_f32(o32, Cout, sd), ref, 3e-3, "tap_sum fp32 output")
        assert o32[..., Cout:].abs().sum().item() == 0
    else:
        temb = torch.randn(N, Cout)
        res = torch.randn_like(ref)
        o = ops.conv(xc, pc, rowvec=temb.cuda(), act1=ops.ACT_SILU, residual=ops.to_cl(res.cuda()))
        ref2 = bf(res) + F.silu(ref + temb.view(N, Cout, *([1] * sd)))
        assert_close(ops.from_cl(o), ref2, 1e-2, "tap_gather conv with fused epilogue")


@pytest.mark.parametrize("impl", [0, 1], ids=IMPL_IDS.get)
def test_conv_groupnorm_partials(cuda_device, monkeypatch, impl):
    """The epilogue's GroupNorm partial sums (b200_igemm gn_partial): per-sample (sum, sumsq) of the stored bf16 outputs
    per 8-channel group, for a plain conv with residual, a 512-channel conv (two 256-column tiles), a two-sample
    batch and the 8-phase upsample conv; then GroupNorm from those partials against the two-pass GroupNorm."""
    ops = _ops()
    monkeypatch.setattr(ops, "_GN_FUSE_MIN_ROWS", 1)
    torch.manual_seed(17)

    def check_partials(out):
        t = out.t.float().cpu()[..., :out.C]                                  # [N, D, H, W, C]
        gw = out.C // out.gn.shape[2]                                         # 8, or 4 for tensors of <= 128 channels
        assert gw == (4 if out.C <= 128 else 8)
        g = t.reshape(t.shape[0], -1, out.C // gw, gw).double()
        want = torch.stack([g.sum((1, 3)), (g * g).sum((1, 3))], -1)        # [N, C/gw, 2]
        got = out.gn.double().sum(1).cpu()
        err = (got - want).abs() / (want.abs() + 1.0)
        assert err.max().item() < 2e-4, err.max().item()

    def gn_both(srcs, groups):
        Ct = sum(a.C for a in srcs)
        g, b = torch.randn(Ct).cuda(), torch.randn(Ct).cuda()
        fused = ops.from_cl(ops.groupnorm(srcs, groups, 1e-6, g, b, act=ops.ACT_SILU))
        monkeypatch.setattr(ops, "_GN_FUSE", False)
        plain = ops.from_cl(ops.groupnorm(srcs, groups, 1e-6, g, b, act=ops.ACT_SILU))
        monkeypatch.setattr(ops, "_GN_FUSE", True)
        assert_close(fused, plain.float().cpu(), 1e-2, "GroupNorm from conv partials vs two-pass")

    x = ops.to_cl(torch.randn(2, 64, 9, 20, 17).cuda())
    mk = lambda co, ci: ops.PackedConv((torch.randn(co, ci, 3, 3, 3) / math.sqrt(ci * 27)).cuda(), torch.randn(co).cuda(), 1, 1)
    res = ops.to_cl(torch.randn(2, 256, 9, 20, 17).cuda())
    a = ops.conv(x, mk(256, 64), rowvec=torch.randn(2, 256).cuda(), act1=ops.ACT_NONE, residual=res, impl=impl)
    b = ops.conv(x, mk(512, 64), impl=impl)
    assert a.gn is not None and b.gn is not None
    check_partials(a)
    check_partials(b)
    gn_both([a], 32)
    gn_both([b, a], 32)           # 768 channels -> groups of 24 spanning 3 producer groups each
    up = ops.conv_upsample2x(a, ops.PackedUpsampleConv((torch.randn(256, 256, 3, 3, 3) / 80).cuda(), torch.randn(256).cuda()), impl=impl)
    check_partials(up)
    gn_both([up], 32)
    # 128 channels: 4-channel partial groups (GroupNorm(32) over 128 channels — level 0 of the 2-D UNets, AutoencoderKL),
    # 128-column tiles; alone, and concatenated with an 8-channel-partial producer
    c = ops.conv(x, mk(128, 64), rowvec=torch.randn(2, 128).cuda(), impl=impl)
    d = ops.conv(x, mk(64, 64), impl=impl)
    assert c.gn is not None and c.gn.shape[2] == 32 and d.gn.shape[2] == 16
    check_partials(c)
    check_partials(d)
    gn_both([c], 32)
    gn_both([a, c], 32)           # 384 channels -> groups of 12: 8-channel partials cannot tile them -> statistics pass
    gn_both([a, c], 48)           # groups of 8: fused from an 8-channel and a 4-channel producer
    gn_both([c, d], 48)           # groups of 4 over two 4-channel producers


def test_conv_asym_pad(cuda_device):
    """AutoencoderKL Downsample: F.pad (0,1) per dim then k3 s2 p0 (autoencoderkl.py:107-120)."""
    ops = _ops()
    for sd, sp in ((2, (16, 18)), (3, (8, 10, 12))):
        x = torch.randn(1, 64, *sp)
        w = torch.randn(64, 64, *([3] * sd)) / math.sqrt(64 * 3 ** sd)
        b = torch.randn(64)
        conv = F.conv2d if sd == 2 else F.conv3d
        ref = conv(F.pad(bf(x), (0, 1) * sd), bf(w), b, stride=2, padding=0)
        pc = ops.PackedConv(w.cuda(), b.cuda(), 2, [(0, 1)] * sd)
        got = ops.from_cl(ops.conv(ops.to_cl(x.cuda()), pc))
        assert tuple(got.shape) == tuple(ref.shape)
        assert_close(got, ref, 1e-2, f"asym-pad conv {sd}d")


@pytest.mark.parametrize("impl", [1, 0], ids=IMPL_IDS.get)
def test_conv_concat_epilogue(cuda_device, impl):
    """Two-source (virtual concat) conv with the full epilogue: bias + temb row vector, SiLU, scale, residual, ReLU."""
    ops = _ops()
    torch.manual_seed(3)
    N, C0, C1, Cout, sp = 2, 64, 32, 96, (6, 10, 12)
    x0, x1 = torch.randn(N, C0, *sp), torch.randn(N, C1, *sp)
    w = torch.randn(Cout, C0 + C1, 3, 3, 3) / math.sqrt((C0 + C1) * 27)
    b = torch.randn(Cout)
    temb = torch.randn(N, Cout)
    res = torch.randn(N, Cout, *sp)
    ref = F.conv3d(torch.cat([bf(x0), bf(x1)], 1), bf(w), b, padding=1) + temb[:, :, None, None, None]
    ref = F.relu(bf(res) + 0.5 * F.silu(ref))
    pc = ops.PackedConv(w.cuda(), b.cuda(), 1, 1, splits=[C0, C1])
    out = ops.conv([ops.to_cl(x0.cuda()), ops.to_cl(x1.cuda())], pc, rowvec=temb.cuda(), act1=ops.ACT_SILU,
                   scale=0.5, residual=ops.to_cl(res.cuda()), act2=ops.ACT_RELU, impl=impl)
    assert_close(ops.from_cl(out), ref, 1e-2, "concat conv + epilogue")
    # batch-broadcast row vector and fp32 output
    out32 = ops.conv([ops.to_cl(x0.cuda()), ops.to_cl(x1.cuda())], pc, rowvec=temb[:1].cuda(), out_f32=True, impl=impl)
    ref32 = F.conv3d(torch.cat([bf(x0), bf(x1)], 1), bf(w), b, padding=1) + temb[:1, :, None, None, None]
    got32 = ops.from_cl_f32(out32, Cout, 3)
    assert_close(got32, ref32, 2e-3, "concat conv fp32 out")


def test_split_k_two_kernel_conv_matches_one_pass_and_check_kernel(cuda_device, monkeypatch):
    """Deep-level shape of a latent UNet (a few hundred voxels, K = 27 x 256): the grid has 2-6 tiles, so the
    reduction is split across the idle SMs and a second kernel applies the epilogue.  Same result as the one-pass
    kernel (fp32 summation order aside) and as the CUDA-core cross-check kernel, for every epilogue option."""
    ops = _ops()
    monkeypatch.setattr(ops, "_SPLIT_K", True)
    torch.manual_seed(11)
    N, Cin, Cout, sp = 2, 256, 200, (5, 7, 5)                     # cout not a multiple of the 64/128 column tile
    x = torch.randn(N, Cin, *sp)
    w = torch.randn(Cout, Cin, 3, 3, 3) / math.sqrt(Cin * 27)
    b, temb, res = torch.randn(Cout), torch.randn(N, Cout), torch.randn(N, Cout, *sp)
    ref = F.conv3d(bf(x), bf(w), b, padding=1) + temb[:, :, None, None, None]
    ref = F.relu(bf(res) + 0.5 * F.silu(ref))
    pc = ops.PackedConv(w.cuda(), b.cuda(), 1, 1)
    xc, rc = ops.to_cl(x.cuda()), ops.to_cl(res.cuda())
    kw = dict(rowvec=temb.cuda(), act1=ops.ACT_SILU, scale=0.5, residual=rc, act2=ops.ACT_RELU)
    n0 = ops._SPLIT_LAUNCHES
    split = ops.from_cl(ops.conv(xc, pc, **kw))
    assert ops._SPLIT_LAUNCHES == n0 + 1, "this shape must take the split-K path"
    monkeypatch.setattr(ops, "_SPLIT_K", False)
    one_pass = ops.from_cl(ops.conv(xc, pc, **kw))
    check = ops.from_cl(ops.conv(xc, pc, impl=1, **kw))
    assert ops._SPLIT_LAUNCHES == n0 + 1
    monkeypatch.setattr(ops, "_SPLIT_K", True)
    assert_close(split, ref, 1e-2, "split-K conv vs torch")
    assert rel_err(split, one_pass)[0] < 2e-3 and rel_err(split, check)[0] < 2e-3, (rel_err(split, one_pass),
                                                                                    rel_err(split, check))
    # strided conv, fp32 output, no epilogue; and determinism of the fixed-order reduction
    pc2 = ops.PackedConv(w.cuda(), None, 2, 1)
    o1 = ops.conv(xc, pc2, out_f32=True)
    o2 = ops.conv(xc, pc2, out_f32=True)
    assert ops._SPLIT_LAUNCHES == n0 + 3 and torch.equal(o1, o2)
    assert_close(ops.from_cl_f32(o1, Cout, 3), F.conv3d(bf(x), bf(w), None, stride=2, padding=1), 2e-3, "split fp32")


def test_split_k_linear_shapes(cuda_device, monkeypatch):
    """GEMM-shaped calls on few rows (transformer blocks of the deepest UNet level): a long feed-forward reduction with a
    residual, and the operand-swapped V^T projection whose bias runs along the rows.  Reductions long enough for the
    planner to split (every range keeps >= 32 chunks of 64)."""
    ops = _ops()
    monkeypatch.setattr(ops, "_SPLIT_K", True)
    torch.manual_seed(12)
    M, K, O = 175, 6144, 768
    x, w, b, r = torch.randn(1, M, K), torch.randn(O, K) / math.sqrt(K), torch.randn(O), torch.randn(1, M, O)
    pl = ops.PackedLinear(w.cuda(), b.cuda())
    xc = ops.as_rows(bf(x).cuda().to(ops.H16), K)
    rc = ops.as_rows(bf(r).cuda().to(ops.H16), O)
    n0 = ops._SPLIT_LAUNCHES
    got = ops.linear(xc, pl, residual=rc)
    assert ops._SPLIT_LAUNCHES == n0 + 1
    ref = F.linear(bf(x), bf(w), b) + bf(r)
    assert_close(got.t.float().cpu().reshape(1, M, -1)[..., :O], ref, 1e-2, "split-K linear + residual")
    xr = bf(torch.randn(2, 200, 6144)).cuda().to(ops.H16)
    w2, b2 = torch.randn(512, 6144) / math.sqrt(6144), torch.randn(512)
    pl2 = ops.PackedLinear(w2.cuda(), b2.cuda())
    vt = ops.linear_transposed(xr, 6144, pl2)                         # [B, O, S_pad]
    assert ops._SPLIT_LAUNCHES == n0 + 2                              # ONE launch for the whole batch (a_broadcast)
    monkeypatch.setattr(ops, "_SPLIT_K", False)
    vt1 = ops.linear_transposed(xr, 6144, pl2)
    ref_vt = (F.linear(xr.float().cpu(), bf(w2), b2)).transpose(1, 2)
    assert_close(vt[..., :200].float().cpu(), ref_vt, 1e-2, "V^T projection")
    assert rel_err(vt.float(), vt1.float())[0] < 2e-3


@pytest.mark.parametrize("sd,sp", [(2, (8, 12)), (3, (4, 6, 8))])
def test_conv_transpose(cuda_device, sd, sp):
    """VQVAE decoder upsampling: ConvTranspose k4 s2 p1 (+ReLU) as per-phase implicit GEMMs (vqvae.py:220-260)."""
    ops = _ops()
    torch.manual_seed(5)
    Cin, Cout = 64, 48
    x = torch.randn(2, Cin, *sp)
    w = torch.randn(Cin, Cout, *([4] * sd)) / math.sqrt(Cin * 2 ** sd)
    b = torch.randn(Cout)
    convt = F.conv_transpose2d if sd == 2 else F.conv_transpose3d
    ref = F.relu(convt(bf(x), bf(w), b, stride=2, padding=1, output_padding=0))
    pt = ops.PackedConvTranspose(w.cuda(), b.cuda(), 2, 1, 0)
    got = ops.from_cl(ops.conv_transpose(ops.to_cl(x.cuda()), pt, act1=ops.ACT_RELU))
    assert tuple(got.shape) == tuple(ref.shape)
    assert_close(got, ref, 1e-2, f"conv_transpose {sd}d")


@pytest.mark.parametrize("sd,sp", [(2, (9, 12)), (3, (5, 6, 8))])
def test_conv_upsample2x(cuda_device, sd, sp):
    """Upsample block: F.interpolate(x2, nearest) + k3 conv as per-phase 2-tap wgmma convolutions."""
    ops = _ops()
    torch.manual_seed(6)
    x = torch.randn(2, 64, *sp)
    w = torch.randn(96, 64, *([3] * sd)) / math.sqrt(64 * 3 ** sd)
    b = torch.randn(96)
    conv = F.conv2d if sd == 2 else F.conv3d
    ref = conv(F.interpolate(bf(x), scale_factor=2.0, mode="nearest"), w, b, padding=1)
    got = ops.from_cl(ops.conv_upsample2x(ops.to_cl(x.cuda()), ops.PackedUpsampleConv(w.cuda(), b.cuda())))
    assert tuple(got.shape) == tuple(ref.shape)
    assert_close(got, ref, 1e-2, f"conv_upsample2x {sd}d")


@pytest.mark.parametrize("M,K,O", [(256, 64, 64), (1000, 320, 512), (77, 40, 24), (4096, 1024, 16), (130, 2048, 256),
                                   (300, 128, 2048), (129, 64, 1100)])
def test_linear(cuda_device, M, K, O):
    ops = _ops()
    torch.manual_seed(M)
    x = torch.randn(1, K, 1, M)          # NCHW with W = rows
    w = torch.randn(O, K) / math.sqrt(K)
    b = torch.randn(O)
    ref = F.linear(bf(x)[0, :, 0].t(), bf(w), b)     # [M, O]
    pl = ops.PackedLinear(w.cuda(), b.cuda())
    out = ops.linear(ops.to_cl(x.cuda()), pl)
    got = out.t[0, 0, 0, :, :O].float().cpu()
    assert_close(got, ref, 1e-2, f"linear {M}x{K}x{O}")


# ------------------------------------------------------------------------------------------------ norms
@pytest.mark.parametrize("shape,groups", [((2, 64, 9, 7), 32), ((1, 256, 6, 10, 12), 32), ((2, 8, 4, 4), 4),
                                            ((1, 96, 5, 5, 5), 32), ((1, 4, 8, 8), 2)])
def test_groupnorm_silu(cuda_device, shape, groups):
    ops = _ops()
    torch.manual_seed(1)
    x = torch.randn(shape) * 2 + 0.5
    g, b = torch.randn(shape[1]), torch.randn(shape[1])
    ref = F.silu(F.group_norm(bf(x), groups, g, b, eps=1e-6))
    out = ops.groupnorm(ops.to_cl(x.cuda()), groups, 1e-6, g.cuda(), b.cuda(), act=ops.ACT_SILU)
    assert_close(ops.from_cl(out), ref, 1e-2, f"groupnorm {shape}")


def test_groupnorm_concat(cuda_device):
    """GroupNorm over a virtual concat whose groups straddle the two tensors (768 = 512 + 256, 24 ch / group)."""
    ops = _ops()
    torch.manual_seed(2)
    x0, x1 = torch.randn(1, 512, 4, 5, 6), torch.randn(1, 256, 4, 5, 6) + 1.0
    g, b = torch.randn(768), torch.randn(768)
    ref = F.group_norm(torch.cat([bf(x0), bf(x1)], 1), 32, g, b, eps=1e-6)
    out = ops.groupnorm([ops.to_cl(x0.cuda()), ops.to_cl(x1.cuda())], 32, 1e-6, g.cuda(), b.cuda())
    assert_close(ops.from_cl(out), ref, 1e-2, "groupnorm concat")


@pytest.mark.parametrize("shape,groups", [((2, 64, 16, 16), 32), ((1, 128, 64, 64), 32), ((2, 32, 5, 7, 5), 8),
                                          ((1, 768, 5, 7, 5), 32), ((2, 24, 9, 11), 8), ((3, 20, 6, 6), 4),
                                          ((1, 12, 33), 12)])
def test_groupnorm_fused_small(cuda_device, monkeypatch, shape, groups):
    """Single-launch GroupNorm (+SiLU) against torch and against the three-kernel path: channel vectors of 8 / 4 / 2 / 1,
    3-D, pad channels, two sources."""
    ops = _ops()
    torch.manual_seed(21)
    if len(shape) == 3:
        shape = (shape[0], shape[1], 1, shape[2])
    x = torch.randn(*shape) * 2 + 0.5
    C_ = shape[1]
    g, b = torch.randn(C_), torch.randn(C_)
    ref = F.silu(F.group_norm(bf(x), groups, g, b, 1e-6))
    xc = ops.to_cl(x.cuda())
    monkeypatch.setattr(ops, "_GN_SMALL", False)
    plain = ops.from_cl(ops.groupnorm(xc, groups, 1e-6, g.cuda(), b.cuda(), act=ops.ACT_SILU))
    monkeypatch.setattr(ops, "_GN_SMALL", True)
    out = ops.groupnorm(xc, groups, 1e-6, g.cuda(), b.cuda(), act=ops.ACT_SILU)
    fused = ops.from_cl(out)
    assert_close(fused, ref, 1e-2, "fused GroupNorm vs torch")
    assert rel_err(fused, plain)[0] < 2e-3
    if out.pitch > C_:
        assert float(out.t[..., C_:].float().abs().max()) == 0.0           # pad channels are exact zeros
    # no activation, and the virtual concat of two sources (groups must not straddle them)
    if C_ % (2 * (C_ // groups)) == 0 and groups % 2 == 0:
        h = C_ // 2
        x0, x1 = ops.to_cl(x[:, :h].contiguous().cuda()), ops.to_cl(x[:, h:].contiguous().cuda())
        cat = ops.from_cl(ops.groupnorm([x0, x1], groups, 1e-6, g.cuda(), b.cuda()))
        assert_close(cat, F.group_norm(bf(x), groups, g, b, 1e-6), 1e-2, "fused GroupNorm over two sources")


def test_layernorm_geglu(cuda_device):
    ops = _ops()
    torch.manual_seed(4)
    M, Cc = 300, 256
    x = torch.randn(1, Cc, 1, M) * 3
    g, b = torch.randn(Cc), torch.randn(Cc)
    ref = F.layer_norm(bf(x)[0, :, 0].t(), (Cc,), g, b, 1e-5)
    out = ops.layernorm(ops.to_cl(x.cuda()), g.cuda(), b.cuda(), 1e-5)
    assert_close(out.t[0, 0, 0, :, :Cc], ref, 1e-2, "layernorm")
    # every width of the 128-bit kernel (1 / 2 / 4 / 8 vectors per lane, ragged last vector) and the scalar fallback
    for C2 in (8, 40, 264, 512, 768, 2048, 12, 2056):
        x2 = torch.randn(1, C2, 1, 67) * 2 + 0.5
        g2, b2 = torch.randn(C2), torch.randn(C2)
        ref2 = F.layer_norm(bf(x2)[0, :, 0].t(), (C2,), g2, b2, 1e-5)
        out2 = ops.layernorm(ops.to_cl(x2.cuda()), g2.cuda(), b2.cuda(), 1e-5)
        assert_close(out2.t[0, 0, 0, :, :C2], ref2, 1e-2, f"layernorm C={C2}")
        assert float(out2.t[0, 0, 0, :, C2:].abs().max() if out2.t.shape[-1] > C2 else 0.0) == 0.0
    xa = bf(x)[0, :, 0].t()
    a, gate = xa.chunk(2, -1)
    refg = a * F.gelu(gate)
    outg = ops.geglu(ops.to_cl(x.cuda()))
    assert_close(outg.t[0, 0, 0, :, : Cc // 2], refg, 1e-2, "geglu")
    # linear1 + gating fused into one GEMM (B200_ACT_GEGLU): grids under and over one wave, a ragged last column tile
    for M2, K2, H2 in ((300, 256, 1024), (32768, 256, 1024), (1000, 64, 160), (70, 512, 2048)):
        x2 = torch.randn(1, K2, 1, M2)
        w2, b2 = torch.randn(2 * H2, K2) / math.sqrt(K2), torch.randn(2 * H2)
        a2, g2 = F.linear(bf(x2)[0, :, 0].t(), bf(w2), b2).chunk(2, -1)
        got = ops.linear_geglu(ops.to_cl(x2.cuda()), ops.PackedLinear.geglu(w2.cuda(), b2.cuda()))
        assert got.C == H2
        assert_close(got.t[0, 0, 0, :, :H2], a2 * F.gelu(g2), 1e-2, f"fused GEGLU linear {M2}x{K2}x{H2}")


# ------------------------------------------------------------------------------------------------ resampling
def test_resample(cuda_device):
    """Through the ops wrappers (layout conversion, pitch, allocation): the F.interpolate / avg_pool / a + alpha b
    checks, bit-exact for avgpool2 (b200_interpolate's AREA sums in fp32 and divides exactly)."""
    from tests import elementwise_emulator as E
    ops = _ops()
    for shape in ((2, 16, 5, 6), (1, 24, 3, 4, 5)):
        x = torch.randn(shape)
        up = ops.from_cl(ops.upsample_nearest2x(ops.to_cl(x.cuda()))).cpu()
        assert torch.equal(up, F.interpolate(bf(x), scale_factor=2.0, mode="nearest"))
    for shape in ((2, 16, 6, 8), (1, 24, 4, 6, 8)):
        x = torch.randn(shape)
        pool = F.avg_pool2d if len(shape) == 4 else F.avg_pool3d
        got = ops.from_cl(ops.avgpool2(ops.to_cl(x.cuda())))
        assert_close(got, pool(bf(x), 2, 2), 1e-2, "avgpool2")
        assert torch.equal(got.cpu().double(), E.h16(pool(bf(x).double(), 2, 2))), "avgpool2 is not bit-exact"
    a, b = torch.randn(1, 16, 4, 4), torch.randn(1, 16, 4, 4)
    got = ops.from_cl(ops.axpy(ops.to_cl(a.cuda()), ops.to_cl(b.cuda()), 0.75))
    assert_close(got, bf(a) + 0.75 * bf(b), 1e-2, "axpy")
    want = E.axpy_h16(a.to(ops.H16).reshape(-1), b.to(ops.H16).reshape(-1), 0.75, a.numel())
    assert E.excess(want, got.cpu().reshape(-1)).max() <= 1, "axpy outside one ulp of fma(alpha, b, a)"


# ------------------------------------------------------------------------------------------------ attention
def _attn_ref(q, k, v, heads, dh, scale):
    B, T, _ = q.shape
    S = k.shape[1]
    qh = q.view(B, T, heads, dh).transpose(1, 2)
    kh = k.view(B, S, heads, dh).transpose(1, 2)
    vh = v.view(B, S, heads, dh).transpose(1, 2)
    p = torch.softmax(scale * qh @ kh.transpose(-1, -2), dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B, T, heads * dh)


@pytest.mark.parametrize("B,T,S,heads,dh", [(2, 64, 64, 2, 4), (1, 16, 16, 1, 8), (2, 100, 3, 1, 256), (1, 50, 1, 2, 64)])
def test_attention_small(cuda_device, B, T, S, heads, dh):
    ops = _ops()
    torch.manual_seed(7)
    Cc = heads * dh
    P = (Cc + 7) // 8 * 8
    q, k, v = torch.randn(B, T, Cc), torch.randn(B, S, Cc), torch.randn(B, S, Cc)
    ref = _attn_ref(bf(q), bf(k), bf(v), heads, dh, 1 / math.sqrt(dh))
    pad = lambda t: F.pad(t, (0, P - Cc)).to(ops.H16).cuda().contiguous()
    out = ops.attention(pad(q), pad(k), pad(v), heads, dh, 1 / math.sqrt(dh))
    assert_close(out[..., :Cc], ref, 1e-2, "attention_small")


@pytest.mark.parametrize("unfused", [False, True], ids=["flash", "unfused"])
@pytest.mark.parametrize("B,T,heads,dh", [(1, 256, 1, 256), (2, 200, 1, 512), (1, 1024, 2, 64), (1, 2300, 1, 128),
                                          (1, 700, 1, 512), (1, 600, 2, 512),
                                          # many query tiles, ragged last tile
                                          (1, 128 * 39 + 50, 1, 512), (2, 128 * 21 + 7, 1, 256)])
def test_attention_tensorcore(cuda_device, B, T, heads, dh, unfused, monkeypatch):
    """Flash-style wgmma attention (scores in registers) and the GEMM + softmax + GEMM path, V^T produced by the
    operand-swapped projection, against fp32 softmax(QK^T)V on the same bf16-rounded q, k, v."""
    ops = _ops()
    monkeypatch.setattr(ops, "_FORCE_UNFUSED_ATTENTION", unfused)
    torch.manual_seed(8)
    Cc = heads * dh
    x = torch.randn(B, T, Cc)
    wq, wk, wv = (torch.randn(Cc, Cc) / math.sqrt(Cc) for _ in range(3))
    bv = torch.randn(Cc)
    xb = bf(x)
    q, k, v = F.linear(xb, bf(wq)), F.linear(xb, bf(wk)), F.linear(xb, bf(wv), bv)
    ref = _attn_ref(bf(q), bf(k), bf(v), heads, dh, 1 / math.sqrt(dh))
    xc = ops.CL(x.to(ops.H16).cuda().reshape(B, 1, 1, T, Cc), Cc, 2)
    plq, plk = ops.PackedLinear(wq.cuda(), None), ops.PackedLinear(wk.cuda(), None)
    plv = ops.PackedLinear(wv.cuda(), bv.cuda())
    qg = ops.linear(xc, plq).t.reshape(B, T, -1)
    kg = ops.linear(xc, plk).t.reshape(B, T, -1)
    vt = ops.linear_transposed(xc.t.reshape(B, T, Cc), Cc, plv)
    assert_close(vt[:, :, :T].transpose(1, 2), bf(v), 1e-2, "V^T projection")
    res = torch.randn(B, T, Cc)
    out = ops.attention(qg, kg, None, heads, dh, 1 / math.sqrt(dh), vt=vt, residual=res.to(ops.H16).cuda())
    assert_close(out[..., :Cc], ref + bf(res), 2e-2, "attention tensor-core")


@pytest.mark.parametrize("dh", [256, 512], ids=["d256", "d512"])
def test_attention_flash_rescale(cuda_device, dh):
    """Keys whose scores grow along the sequence raise the running row maximum by large factors many times, exercising
    the online-softmax rescale of the output accumulator (for head_dim 512 in both 256-channel output slices)."""
    ops = _ops()
    torch.manual_seed(11)
    B, T, S = 1, 128 * 40 + 9, 1000
    q = torch.randn(B, T, dh)
    k = torch.randn(B, S, dh) * torch.linspace(0.2, 9.0, S)[None, :, None]
    v = torch.randn(B, S, dh)
    scale = 1 / math.sqrt(dh)
    ref = _attn_ref(bf(q), bf(k), bf(v), 1, dh, scale)
    vt = v.to(ops.H16).transpose(1, 2).contiguous().cuda()
    out = ops.attention(q.to(ops.H16).cuda(), k.to(ops.H16).cuda(), None, 1, dh, scale, vt=vt)
    assert_close(out[..., :dh], ref, 2e-2, "flash attention with rescale")


def test_attention_flash_d512_ragged_batches(cuda_device):
    """head_dim 512 (two 256-channel output slices per query tile, each recomputing the scores) on a multi-batch,
    ragged problem (T, S not multiples of the tiles; more work items than SMs) with late rescales and a residual: every
    row and both output slices of both batches against the fp32 reference."""
    ops = _ops()
    torch.manual_seed(12)
    B, T, S, dh = 2, 128 * 90 + 37, 1000 + 21, 512
    q, k, v = torch.randn(B, T, dh), torch.randn(B, S, dh), torch.randn(B, S, dh)
    k[:, 500:] *= 6.0                                     # the running maximum jumps late in many rows
    res = torch.randn(B, T, dh).to(ops.H16).cuda()
    args = (q.to(ops.H16).cuda(), k.to(ops.H16).cuda(), None, 1, dh, 1 / math.sqrt(dh))
    vt = F.pad(v.to(ops.H16).transpose(1, 2), (0, (-S) % 8)).contiguous().cuda()
    a = ops.attention(*args, vt=vt, residual=res).float().cpu()
    ref = _attn_ref(bf(q), bf(k), bf(v), 1, dh, 1 / math.sqrt(dh)) + res.float().cpu()
    for b in range(B):
        for lo in (0, 256):
            assert_close(a[b, :, lo:lo + 256], ref[b, :, lo:lo + 256], 2e-2, f"batch {b}, channels {lo}..{lo + 255}")


@pytest.mark.parametrize("B,T,S,heads,dh,q_pos0,causal", [(2, 9, 9, 4, 8, 0, True), (3, 1, 37, 2, 64, 36, True),
                                                          (1, 5, 20, 1, 32, 15, True), (2, 6, 11, 2, 16, 0, False)])
def test_attention_causal_and_cache(cuda_device, B, T, S, heads, dh, q_pos0, causal):
    """b200_attention_small_ex: causal mask by absolute position and keys / values living in a longer cache
    (SABlock, blocks/selfattention.py:121-140; the decode step of the transformer sampler)."""
    ops = _ops()
    torch.manual_seed(21)
    Cc = heads * dh
    rows = S + 5                                             # cache longer than the valid prefix
    q, k, v = torch.randn(B, T, Cc), torch.randn(B, rows, Cc), torch.randn(B, rows, Cc)
    qh = bf(q).view(B, T, heads, dh).transpose(1, 2)
    kh = bf(k)[:, :S].reshape(B, S, heads, dh).transpose(1, 2)
    vh = bf(v)[:, :S].reshape(B, S, heads, dh).transpose(1, 2)
    sc = (qh @ kh.transpose(-1, -2)) / math.sqrt(dh)
    if causal:
        allowed = torch.arange(S)[None, :] <= (q_pos0 + torch.arange(T))[:, None]
        sc = sc.masked_fill(~allowed, float("-inf"))
    ref = (torch.softmax(sc, -1) @ vh).transpose(1, 2).reshape(B, T, Cc)
    g = lambda t: t.to(ops.H16).cuda().contiguous()
    out = ops.attention_causal(g(q), g(k), g(v), heads, dh, 1 / math.sqrt(dh), S, causal=causal, q_pos0=q_pos0)
    assert_close(out[..., :Cc], ref, 1e-2, "causal attention over a cache")


def test_embed_tokens_gelu_and_cache_projection(cuda_device):
    """Token + position embedding rows, exact-erf GELU in the GEMM epilogue, and the K / V projection that writes
    its rows straight into a [B, max_seq, C] cache at an offset (nets/transformer.py:97-99; MLPBlock)."""
    ops = _ops()
    torch.manual_seed(22)
    B, T, C_, V, L = 3, 5, 40, 17, 12
    tok, pos = torch.randn(V, C_), torch.randn(L, C_)
    x = torch.randint(0, V, (B, T))
    e = ops.embed_tokens(x.cuda(), tok.cuda(), pos.cuda(), pos0=4)
    want = tok[x] + pos[4 + torch.arange(T)][None]
    assert_close(e.t.reshape(B, T, -1)[..., :C_], want, 1e-2, "embed_tokens")
    assert e.t.reshape(B * T, -1)[:, C_:].abs().sum().item() == 0
    w, b = torch.randn(64, C_) / math.sqrt(C_), torch.randn(64)
    pl = ops.PackedLinear(w.cuda(), b.cuda())
    y = ops.linear(e, pl, act1=ops.ACT_GELU)
    assert_close(y.t.reshape(B * T, -1)[:, :64], F.gelu(F.linear(bf(want).reshape(B * T, C_), bf(w), b)), 1e-2, "GELU epilogue")
    cache = torch.zeros(B, L, 64, dtype=ops.H16, device="cuda")
    ops.linear_into_cache(e, B, T, pl, cache, 6)
    lin = F.linear(bf(want), bf(w), b)
    assert_close(cache[:, 6:6 + T], lin, 1e-2, "projection into the cache")
    assert cache[:, :6].abs().sum().item() == 0 and cache[:, 6 + T:].abs().sum().item() == 0


@pytest.mark.parametrize("M,K,O,ln,act,res,f32out", [(1, 512, 512, True, 0, False, False), (8, 512, 2048, True, 4, False, False),
                                                     (3, 2048, 512, False, 0, True, False), (2, 40, 257, False, 0, False, True),
                                                     (5, 64, 17, True, 2, True, False)])
def test_rows_linear(cuda_device, M, K, O, ln, act, res, f32out):
    """b200_rows_linear: decode-time GEMV with LayerNorm prologue and bias / activation / residual epilogue."""
    ops = _ops()
    torch.manual_seed(23)
    x, w, b = torch.randn(M, K), torch.randn(O, K) / math.sqrt(K), torch.randn(O)
    g, be = torch.randn(K), torch.randn(K)
    r = torch.randn(M, O)
    xin = bf(x)
    if ln:
        xin = bf(F.layer_norm(xin, (K,), g, be, 1e-5))
    ref = F.linear(xin, bf(w), b)
    ref = {0: ref, 2: F.silu(ref), 4: F.gelu(ref)}[act]
    if res:
        ref = ref + bf(r)
    P = (K + 7) // 8 * 8
    xg = F.pad(x, (0, P - K)).to(ops.H16).cuda()
    pl = ops.PackedLinear(w.cuda(), b.cuda())
    rg = F.pad(r, (0, (-O) % 8)).to(ops.H16).cuda() if res else None
    out = ops.rows_linear(xg, K, pl, ln=(g.cuda(), be.cuda(), 1e-5) if ln else None, act=act, residual=rg, out_f32=f32out)
    assert out.dtype == (torch.float32 if f32out else ops.H16)
    assert_close(out[:, :O], ref, 1e-2, "rows_linear")


@pytest.mark.parametrize("B,S,heads,dh", [(1, 1, 8, 64), (3, 1000, 8, 64), (8, 37, 2, 32), (2, 300, 1, 256)])
def test_attention_decode(cuda_device, B, S, heads, dh):
    """b200_attention_decode (keys split over 8 warps, merged online-softmax states) incl. the device-side length."""
    ops = _ops()
    torch.manual_seed(24)
    Cc = heads * dh
    rows = S + 3
    q, k, v = torch.randn(B, Cc), torch.randn(B, rows, Cc), torch.randn(B, rows, Cc)
    ref = _attn_ref(bf(q)[:, None], bf(k)[:, :S], bf(v)[:, :S], heads, dh, 1 / math.sqrt(dh))[:, 0]
    g = lambda t: t.to(ops.H16).cuda().contiguous()
    out = ops.attention_decode(g(q), g(k), g(v), heads, dh, 1 / math.sqrt(dh), S)
    assert_close(out[:, :Cc], ref, 1e-2, "attention_decode")
    pos = torch.tensor([S - 1], dtype=torch.int32).cuda()
    out2 = ops.attention_decode(g(q), g(k), g(v), heads, dh, 1 / math.sqrt(dh), 1, pos_dev=pos)
    assert torch.equal(out, out2)


# ------------------------------------------------------------------------------------------------ time embedding
def test_timestep_embedding_and_small_linear(cuda_device):
    """Through the ops wrappers: the fp32 restatements, and the contract of tests/elementwise_emulator.py on top."""
    from tests import elementwise_emulator as E
    ops = _ops()
    t = torch.tensor([0.0, 1.0, 250.0, 999.0])
    for dim in (32, 33, 256):
        half = dim // 2
        exponent = -math.log(10000) * torch.arange(0, half, dtype=torch.float32)
        freqs = torch.exp(exponent / half)
        args = t[:, None] * freqs[None]
        ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
        if dim % 2:
            ref = F.pad(ref, (0, 1))
        got = ops.timestep_embedding(t.cuda(), dim).cpu()
        assert (got - ref).abs().max().item() < 2e-4
        assert E.excess(E.timestep_embedding(t, 4, dim, 10000.0), got).max() <= 1, dim
    x = torch.randn(3, 100)
    w, b = torch.randn(70, 100) / 10, torch.randn(70)
    ref = F.silu(F.linear(F.silu(x), w, b))
    got = ops.small_linear(x.cuda(), w.cuda(), b.cuda(), ops.ACT_SILU, ops.ACT_SILU).cpu()
    assert (got - ref).abs().max().item() < 1e-4
    want = E.small_linear(x.reshape(-1), 3, 100, w.reshape(-1), b, 70, E.ACT_SILU, E.ACT_SILU)
    assert E.excess(want, got).max() <= 1
    for K in (1024, 384, 2176):                    # K % 128 == 0: the float4 path (one / partial / three 1024-blocks)
        x = torch.randn(2, K)
        w, b = torch.randn(300, K) / math.sqrt(K), torch.randn(300)
        ref = F.linear(F.silu(x), w, b)
        got = ops.small_linear(x.cuda(), w.cuda(), b.cuda(), ops.ACT_SILU, ops.ACT_NONE).cpu()
        assert (got - ref).abs().max().item() < 1e-4, K
        want = E.small_linear(x.reshape(-1), 2, K, w.reshape(-1), b, 300, E.ACT_SILU, E.ACT_NONE)
        assert E.excess(want, got).max() <= 1, K


# ------------------------------------------------------------------------------------------------ perf smoke (prints)
def test_conv_perf_probe(cuda_device, capsys):
    """Not a benchmark: one warm conv at a C3-like tile mix to catch gross slowness early (printed with -s)."""
    ops = _ops()
    x = torch.randn(1, 256, 16, 112, 80)
    w = torch.randn(256, 256, 3, 3, 3) / 80
    pc = ops.PackedConv(w.cuda(), None, 1, 1)
    a = ops.to_cl(x.cuda())
    for _ in range(2):
        ops.conv(a, pc)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        ops.conv(a, pc)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 5
    flops = 2 * 16 * 112 * 80 * 256 * 256 * 27
    with capsys.disabled():
        print(f"\n[perf-probe] conv3d 256->256 k3 @16x112x80: {ms:.3f} ms, {flops / ms / 1e9:.1f} TFLOP/s")
    assert ms > 0


def test_repack_weight_matches_host_restatement(cuda_device, monkeypatch):
    """b200_repack_weight (one launch per weight) against the literal host restatement in tests/cpu_backend.py, bit for
    bit: plain / split (virtual concat) / strided convolutions, linear, the folded-upsample phase sums (2-D and 3-D),
    transposed-convolution phases and the two degenerate tap reformulations."""
    from tests import cpu_backend
    torch.manual_seed(0)
    r = torch.randn
    cases = [
        ("conv3d", r(96, 72, 3, 3, 3), lambda w: ops.PackedConv(w, None, 1, 1)),
        ("conv3d split", r(96, 72, 3, 3, 3), lambda w: ops.PackedConv(w, None, 1, 1, splits=[40, 32])),
        ("conv2d stride 2", r(130, 200, 3, 3), lambda w: ops.PackedConv(w, None, 2, 1)),
        ("conv k4", r(64, 32, 4, 4, 4), lambda w: ops.PackedConv(w, None, 2, 1)),
        ("conv_in (tap_in)", r(256, 1, 3, 3, 3), lambda w: ops.PackedConv(w, None, 1, 1)),
        ("out conv (tap_out)", r(1, 256, 3, 3, 3), lambda w: ops.PackedConv(w, None, 1, 1)),
        ("linear", r(300, 520), lambda w: ops.PackedLinear(w, None)),
        ("upsample 3d", r(64, 72, 3, 3, 3), lambda w: ops.PackedUpsampleConv(w, None)),
        ("upsample 2d", r(48, 130, 3, 3), lambda w: ops.PackedUpsampleConv(w, None)),
        ("convT 3d", r(72, 40, 4, 4, 4), lambda w: ops.PackedConvTranspose(w, None, 2, 1, 0)),
        ("convT 2d", r(64, 24, 4, 4), lambda w: ops.PackedConvTranspose(w, None, 2, 1, 0)),
    ]

    def mats(p):
        out = [ph[1] for ph in p.phases] if hasattr(p, "phases") else [p.w]
        for extra in ("tap_in", "tap_out"):
            if getattr(p, extra, None) is not None:
                out.append(getattr(p, extra).w)
        return out

    for name, w, build in cases:
        with monkeypatch.context() as mp:
            cpu_backend.install(mp)
            want = [m.clone() for m in mats(build(w))]
        got = mats(build(w.cuda()))
        assert len(got) == len(want), name
        for g, x in zip(got, want):
            assert g.is_cuda and g.shape == x.shape and g.dtype == x.dtype, name
            assert torch.equal(g.cpu().view(torch.int16), x.view(torch.int16)), f"{name}: packed weights differ"

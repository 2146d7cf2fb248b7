"""The checks of tests/test_gn_partials_gpu.py verified without a GPU: the convolutions and GroupNorms of ops run through
the CPU stand-in of the C ABI (tests/cpu_backend.py, whose b200_igemm is tests/igemm_emulator.py: it writes the
GroupNorm partials of the stored values in one slot), and the float64 reference (tests/gn_partials_reference.py) must
accept them; then four broken producers, each one slip a kernel's epilogue could make, must be rejected:

  slot_off_by_one     the slot index one too far: the last slot of a sample lands in the next sample's first
  width_mixup         8-channel group sums written into the 4-channel layout the consumer reads
  no_final_flush      each warp's last work item never reaches its slot
  fp32_accumulator    sums of the fp32 values before the 16-bit rounding instead of the stored values

The producers deal the rows to slots as the kernels do: 128-row work items round robin over the CTAs, 32 rows of each
to each of a CTA's four slots, one fp32 add per item.
"""
import math
import zlib

import pytest
import torch

from generativemodels_b200 import ops
from tests import cpu_backend
from tests import gn_partials_reference as R

SM = 2                           # the stand-in's b200_sm_count


@pytest.fixture
def fake(monkeypatch):
    cpu_backend.install(monkeypatch)
    monkeypatch.setattr(ops, "_SM_COUNT", None)
    monkeypatch.setattr(ops, "_GN_FUSE_MIN_ROWS", 1)       # small grids: the rule is the networks', not the check's
    yield


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


def cl(g, N, dims, C, sd):
    return ops.CL(torch.randn(N, *dims, C, generator=g).to(ops.H16), C, sd)


def packed(g, cout, cin, sd, k, group_offsets, groups):
    """3^sd convolution, weights ~ N(0, 1/fan_in); the bias puts k standard deviations of offset on every group, with a
    sign per group."""
    w = torch.randn(cout, cin, *([3] * sd), generator=g) / math.sqrt(cin * 3 ** sd)
    sign = torch.where(torch.rand(groups, generator=g) < 0.5, -1.0, 1.0).repeat_interleave(cout // groups)
    return ops.PackedConv(w, k * sign + 0.1 * torch.randn(cout, generator=g) if group_offsets else None, 1, 1)


def affine_args(g, C):
    return 1 + 0.5 * torch.randn(C, generator=g), 0.5 * torch.randn(C, generator=g)


def run(srcs, groups, prod, g):
    gamma, beta = affine_args(g, sum(a.C for a in srcs))
    assert R.takes_partials(srcs, groups)
    table = ops.groupnorm_affine(srcs, groups, 1e-6, gamma, beta)
    return R.check(srcs, groups, 1e-6, gamma, beta, table, [prod.of(a) for a in srcs])


CASES = ["conv2d_c32_g8", "conv3d_c256_residual", "upsample2d_c128", "concat2d_128_128"]


@pytest.mark.parametrize("k", [0.0, 3.0, 30.0], ids=lambda k: f"k{int(k)}")
@pytest.mark.parametrize("case", CASES)
def test_reference_accepts_the_emulated_producer(fake, case, k):
    g = gen(f"{case}/{k}")
    with R.Producers(SM) as prod:
        if case == "conv2d_c32_g8":
            out, groups = ops.conv(cl(g, 2, (1, 12, 20), 32, 2), packed(g, 32, 32, 2, k, True, 8)), 8
            srcs = [out]
        elif case == "conv3d_c256_residual":
            x, res = cl(g, 1, (3, 4, 5), 64, 3), cl(g, 1, (3, 4, 5), 256, 3)
            srcs, groups = [ops.conv(x, packed(g, 256, 64, 3, k, True, 32), residual=res)], 32
        elif case == "upsample2d_c128":
            x = cl(g, 1, (1, 6, 7), 64, 2)
            w = torch.randn(128, 64, 3, 3, generator=g) / 24
            bias = k * torch.where(torch.rand(32, generator=g) < 0.5, -1.0, 1.0).repeat_interleave(4)
            srcs, groups = [ops.conv_upsample2x(x, ops.PackedUpsampleConv(w, bias))], 32
        else:
            x = cl(g, 2, (1, 8, 8), 32, 2)
            srcs = [ops.conv(x, packed(g, 128, 32, 2, k, True, 32)), ops.conv(x, packed(g, 128, 32, 2, k, True, 32))]
            groups = 32
    r = run(srcs, groups, prod, g)
    print(f"\nGN-PARTIALS cpu {case} k={k:g}: {R.fmt(r)}")
    assert r.contract <= 1 and r.product <= 1 and r.totals <= 1, R.fmt(r)


# ------------------------------------------------------------------------------------------------------------------
# producers with the kernels' slot layout, and four ways to break them
# ------------------------------------------------------------------------------------------------------------------
def kernel_partials(values, gw, slots, mutant=None):
    """[N, S, C] float64 output values -> fp32 partials [N, slots, C / gw, 2], rows dealt as the kernels deal them."""
    Nn, S, Cc = values.shape
    width = 8 if mutant == "width_mixup" else gw
    items = [(n, r0) for n in range(Nn) for r0 in range(0, S, 128)]
    ctas = min(len(items), SM)
    flat = torch.zeros(Nn * slots * (Cc // gw) * 2, dtype=torch.float32)
    for cta in range(ctas):
        mine = items[cta::ctas]
        for warp in range(4):
            for i, (n, r0) in enumerate(mine):
                if mutant == "no_final_flush" and i == len(mine) - 1:
                    continue
                v = values[n, r0 + 32 * warp:r0 + 32 * warp + 32].reshape(-1, Cc // width, width)
                add = torch.stack([v.sum((0, 2)), (v * v).sum((0, 2))], -1).float().reshape(-1)
                slot = n * slots + 4 * cta + warp + (1 if mutant == "slot_off_by_one" else 0)
                if slot >= Nn * slots:
                    continue
                base = slot * (Cc // width) * 2      # the mix-up also strides the slots by the wrong group count
                flat[base:base + add.numel()] += add
    return flat.view(Nn, slots, Cc // gw, 2)


MUTANTS = ["slot_off_by_one", "width_mixup", "no_final_flush", "fp32_accumulator"]


@pytest.mark.parametrize("mutant", [None, *MUTANTS], ids=lambda m: m or "faithful")
def test_bound_rejects_broken_producers(fake, mutant):
    """16 x 16 voxels of 2 samples, 128 channels (4-channel partial groups), k = 3: every slot of both CTAs receives
    rows of two work items."""
    g = gen("mutants")
    x = cl(g, 2, (1, 16, 16), 32, 2)
    pc = packed(g, 128, 32, 2, 3.0, True, 32)
    with R.Producers(SM) as prod:
        out = ops.conv(x, pc)
    assert ops._gn_group(out) == 4 and out.gn.shape[1] == 4 * SM
    stored = out.t.view(2, -1, out.pitch)[..., :128].double()
    values = ops.conv(x, pc, out_f32=True).view(2, -1, 128).double() if mutant == "fp32_accumulator" else stored
    out.gn.copy_(kernel_partials(values, 4, out.gn.shape[1], mutant))
    r = run([out], 32, prod, g)
    worst = max(r.contract, r.totals)
    print(f"\nGN-PARTIALS mutant {mutant or 'faithful'}: {R.fmt(r)}  rejected by x{worst:.3g}")
    if mutant is None:
        assert r.contract <= 1 and r.product <= 1 and r.totals <= 1, R.fmt(r)
    else:
        assert worst > 1, f"{mutant} passes the bound: {R.fmt(r)}"

"""GroupNorm fed by the partial sums of b200_igemm's epilogue, through ops the way the networks call it, against the
float64 reference of tests/gn_partials_reference.py: the stored h16 output of the producing convolution(s) read back,
per-(sample, group) moments in float64, the affine table by norm_emulator's formula.  Every table is held to

  contract  the header's from-partials bound, T = terms per fp32 slot from the launch's tile plan (must always hold);
  product   the bound b200_groupnorm_stats is held to (2^-12 against the group's pivot), at every offset of the sweep
            and every call of the networks;
  totals    slot totals = float64 sums of the stored values, within the rounding depth of the epilogue's summation.

The producer sweep covers 2-D and 3-D, 4- and 8-channel partial groups, the 128-column and the two-CTA kernel, the
residual epilogue, conv_upsample2x (one launch per phase, slot ranges from gn_slot0), a two-source GroupNorm, N = 1-3,
from about one work item per slot to over a hundred, and per-group offsets k |mean| / std in {0, 1, 3, 10, 30, 100}
set through the bias.  The network tests wrap ops.groupnorm_affine and check every call that takes the path.  Lines
starting GN-PARTIALS report k and err / tol.
"""
import math
import zlib
from dataclasses import dataclass

import pytest
import torch

from generativemodels_b200 import ops
from tests import gn_partials_reference as R
from tests import golden
from tests.golden import configs as G

pytestmark = pytest.mark.gpu

EPS = 1e-6
K_VALUES = (0.0, 1.0, 3.0, 10.0, 30.0, 100.0)


def gen(name):
    return torch.Generator().manual_seed(zlib.crc32(name.encode()))


@pytest.fixture(scope="module")
def sm(cuda_device):
    return int(ops._lib.require_device().b200_sm_count())


def randn(g, *shape):
    return torch.randn(*shape, generator=g).cuda()


def cl(g, N, dims, C, sd):
    return ops.CL(randn(g, N, *dims, C).to(ops.H16), C, sd)


def group_bias(g, cout, groups, k):
    """k standard deviations of offset on every group (sign per group) plus a little per-channel spread."""
    sign = torch.where(torch.rand(groups, generator=g) < 0.5, -1.0, 1.0).repeat_interleave(cout // groups)
    return (k * sign + 0.1 * torch.randn(cout, generator=g)).cuda()


@dataclass(frozen=True)
class Prod:
    name: str
    sd: int
    N: int
    dims: tuple          # output extent (the source's for an upsample)
    C: int
    cin: int
    groups: int
    impl: int = 0        # 0 planner, 2 the 128-column kernel, 3 the two-CTA kernel
    kind: str = "conv"   # conv / residual / upsample / concat (a second producer of C1 channels)
    C1: int = 0


PRODUCERS = [
    Prod("2d_c32_g8_n1_min_rows", 2, 1, (1, 184, 184), 32, 32, 8, impl=2),
    Prod("2d_c64_g16_n3", 2, 3, (1, 128, 128), 64, 64, 16),
    Prod("2d_c128_n2_residual", 2, 2, (1, 128, 128), 128, 128, 32, kind="residual"),
    Prod("2d_c160_g20", 2, 1, (1, 256, 256), 160, 64, 20),
    Prod("2d_c512_wide_residual", 2, 1, (1, 256, 256), 512, 128, 32, impl=3, kind="residual"),
    Prod("3d_c32_g8_128col_large", 3, 1, (120, 120, 120), 32, 32, 8, impl=2),
    Prod("3d_c256_128col_n3", 3, 3, (40, 40, 40), 256, 64, 32, impl=2),
    Prod("3d_c256_wide_n2", 3, 2, (32, 40, 32), 256, 256, 32, impl=3),
    Prod("3d_c512_wide_large", 3, 1, (96, 96, 96), 512, 64, 32, impl=3),
    Prod("2d_upsample_c128", 2, 1, (1, 192, 192), 128, 128, 32, kind="upsample"),
    Prod("3d_upsample_c256", 3, 1, (32, 32, 32), 256, 256, 32, kind="upsample"),
    Prod("2d_concat_128_128_n2", 2, 2, (1, 128, 128), 128, 64, 32, kind="concat", C1=128),
    Prod("3d_concat_256_256", 3, 1, (40, 56, 40), 256, 64, 32, kind="concat", C1=256),
]


def weights(g, cout, cin, sd):
    return randn(g, cout, cin, *([3] * sd)) / math.sqrt(cin * 3 ** sd)


@pytest.mark.parametrize("c", PRODUCERS, ids=[c.name for c in PRODUCERS])
def test_producer_sweep(sm, c):
    g = gen(c.name)
    x = cl(g, c.N, c.dims, c.cin, c.sd)
    res = cl(g, c.N, c.dims, c.C, c.sd) if c.kind == "residual" else None
    w = weights(g, c.C, c.cin, c.sd)
    w1 = weights(g, c.C1, c.cin, c.sd) if c.C1 else None
    Ct = c.C + c.C1
    gamma, beta = (1 + 0.5 * torch.randn(Ct, generator=g)).cuda(), (0.5 * torch.randn(Ct, generator=g)).cuda()
    cpg = Ct // c.groups
    rows = []
    for k in K_VALUES:
        with R.Producers(sm) as prod:
            if c.kind == "upsample":
                srcs = [ops.conv_upsample2x(x, ops.PackedUpsampleConv(w, group_bias(g, c.C, c.C // cpg, k)))]
            else:
                srcs = [ops.conv(x, ops.PackedConv(w, group_bias(g, c.C, c.C // cpg, k), 1, 1), residual=res,
                                 impl=c.impl)]
                if c.C1:
                    srcs.append(ops.conv(x, ops.PackedConv(w1, group_bias(g, c.C1, c.C1 // cpg, k), 1, 1),
                                         impl=c.impl))
        assert R.takes_partials(srcs, c.groups), f"{c.name}: the GroupNorm does not read the convolution's partials"
        table = ops.groupnorm_affine(srcs, c.groups, EPS, gamma, beta)
        r = R.check(srcs, c.groups, EPS, gamma, beta, table, [prod.of(a) for a in srcs])
        print(f"\nGN-PARTIALS producer {c.name} k={k:g}: {R.fmt(r)}")
        rows.append((k, r))
        del srcs, table
    for k, r in rows:
        assert r.contract <= 1, f"{c.name} k={k:g}: outside the header's from-partials bound: {R.fmt(r)}"
        assert r.totals <= 1, f"{c.name} k={k:g}: slot totals are not sums of the stored values: {R.fmt(r)}"
        assert r.product <= 1, f"{c.name} k={k:g}: outside the statistics pass's bound: {R.fmt(r)}"


def _step(x, pc, res, gamma, beta, groups):
    out = ops.conv(x, pc, residual=res)
    return ops.groupnorm_affine(out, groups, EPS, gamma, beta)


@pytest.mark.parametrize("sd,N,dims,C,cin", [(3, 2, (32, 40, 32), 256, 256), (2, 2, (1, 128, 128), 128, 128)],
                         ids=["3d_c256_planner", "2d_c128"])
def test_tables_bit_identical_repeated_and_graph_replayed(sm, sd, N, dims, C, cin):
    g = gen(f"determinism/{sd}")
    x, res = cl(g, N, dims, cin, sd), cl(g, N, dims, C, sd)
    pc = ops.PackedConv(weights(g, C, cin, sd), group_bias(g, C, 32, 3.0), 1, 1)
    gamma, beta = (1 + 0.5 * torch.randn(C, generator=g)).cuda(), (0.5 * torch.randn(C, generator=g)).cuda()
    eager = [_step(x, pc, res, gamma, beta, 32).clone() for _ in range(3)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _step(x, pc, res, gamma, beta, 32)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        table = _step(x, pc, res, gamma, beta, 32)
    replays = []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        replays.append(table.clone())
    for t in eager[1:] + replays:
        assert torch.equal(t.view(torch.int32), eager[0].view(torch.int32)), "affine table differs between runs"


# ------------------------------------------------------------------------------------------------------------------
# the networks
# ------------------------------------------------------------------------------------------------------------------
BRAIN_AE = dict(spatial_dims=3, in_channels=1, out_channels=1, latent_channels=3, num_channels=(64, 128, 128, 128),
                num_res_blocks=2, norm_num_groups=32, norm_eps=1e-06, attention_levels=(False,) * 4,
                with_encoder_nonlocal_attn=False, with_decoder_nonlocal_attn=False)
BRAIN_UNET = dict(spatial_dims=3, in_channels=7, out_channels=3, num_channels=(256, 512, 768), num_res_blocks=2,
                  attention_levels=(False, True, True), norm_num_groups=32, norm_eps=1e-06, resblock_updown=True,
                  num_head_channels=(0, 512, 768), with_conditioning=True, transformer_num_layers=1,
                  cross_attention_dim=4, upcast_attention=True, use_flash_attention=False)
C3_VOLUME = (160, 224, 160)      # bench.py's flagship volume


def _net(name):
    """(module on the GPU with recipe weights, forward closure, whether any GroupNorm input is large enough to take
    the path: >= 2^15 rows and a heavy producer)."""
    from generativemodels_b200.networks.nets import AutoencoderKL, DiffusionModelUNet
    g = gen(name)
    if name == "c3_unet_full":
        m = DiffusionModelUNet(**G.C3_UNET)
        G.recipe_state_dict(m, 13)
        x = torch.randn(1, 1, *C3_VOLUME, generator=g)
        return m, lambda m: m(x.cuda(), timesteps=torch.tensor([500.0]).cuda()), True
    if name == "c5_unet_cfg_batch":
        m = DiffusionModelUNet(**G.C5_UNET)
        G.recipe_state_dict(m, 5)
        x, ctx = torch.randn(2, *G.C5_SHAPE[1:], generator=g), torch.randn(2, 1, 1, generator=g)
        return m, lambda m: m(x.cuda(), timesteps=torch.tensor([480.0, 480.0]).cuda(), context=ctx.cuda()), True
    if name == "brain_ldm_unet":
        m = DiffusionModelUNet(**BRAIN_UNET)
        G.recipe_state_dict(m, 7)
        x, ctx = torch.randn(1, 7, 20, 28, 20, generator=g), torch.randn(1, 1, 4, generator=g)
        return m, lambda m: m(x.cuda(), timesteps=torch.tensor([500.0]).cuda(), context=ctx.cuda()), False
    if name == "brain_ldm_decoder":
        m = AutoencoderKL(**BRAIN_AE)
        G.recipe_state_dict(m, 11)
        z = torch.randn(1, 3, 20, 28, 20, generator=g)
        return m, lambda m: m.decode(z.cuda()), True
    fx = golden.load("g_bundle_mednist_ddpm")
    m = DiffusionModelUNet(**fx["unet_kwargs"])
    G.recipe_state_dict(m, fx["unet_seed"])
    x = torch.randn(1, 1, 64, 64, generator=g)
    return m, lambda m: m(x.cuda(), timesteps=torch.tensor([500.0]).cuda()), False


NETWORKS = ["c3_unet_full", "c5_unet_cfg_batch", "brain_ldm_unet", "brain_ldm_decoder", "mednist_unet"]


@pytest.mark.parametrize("name", NETWORKS)
def test_networks(sm, monkeypatch, name):
    m, forward, expect_calls = _net(name)
    m = m.cuda().eval()
    reports = []
    orig = ops.groupnorm_affine

    def checked(srcs, groups, eps, gamma, beta):
        table = orig(srcs, groups, eps, gamma, beta)
        s = [srcs] if isinstance(srcs, ops.CL) else list(srcs)
        if R.takes_partials(s, groups):
            reports.append(R.check(s, groups, eps, gamma, beta, table, [prod.of(a) for a in s]))
        return table

    monkeypatch.setattr(ops, "groupnorm_affine", checked)
    with torch.no_grad(), R.Producers(sm) as prod:
        forward(m)
    torch.cuda.synchronize()
    if not reports:
        print(f"\nGN-PARTIALS network {name}: no GroupNorm reads convolution partials")
        assert not expect_calls, f"{name}: expected GroupNorms fed by convolution partials, found none"
        return
    worst = lambda f: max(reports, key=f)
    print(f"\nGN-PARTIALS network {name}: {len(reports)} calls; largest k {worst(lambda r: r.k).k:.2f}, "
          f"work/slot {worst(lambda r: r.work_per_slot).work_per_slot}; err/tol contract "
          f"{worst(lambda r: r.contract).contract:.3g} product {worst(lambda r: r.product).product:.3g} totals "
          f"{worst(lambda r: r.totals).totals:.3g}")
    for i, r in enumerate(reports):
        assert r.contract <= 1 and r.totals <= 1 and r.product <= 1, f"{name}: GroupNorm call {i}: {R.fmt(r)}"
